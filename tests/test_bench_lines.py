"""bench.py's argument surface.  CPU only: nothing here runs the hot path."""
import ast
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_bench_argument_surface():
    """--gpus / --steps / --warmup / --impl / --dump-outputs exist with the expected defaults (N=1, W >= 3)"""
    tree = ast.parse(open(os.path.join(ROOT, "bench.py")).read())
    args = {}
    for node in ast.walk(tree):
        if isinstance(node, ast.Call) and getattr(node.func, "attr", "") == "add_argument" and node.args:
            name = node.args[0].value if isinstance(node.args[0], ast.Constant) else None
            kw = {k.arg: k.value for k in node.keywords}
            default = kw.get("default")
            args[name] = default.value if isinstance(default, ast.Constant) else None
    assert {"--gpus", "--steps", "--warmup", "--impl", "--dump-outputs"} <= set(args)
    assert args["--gpus"] == 1 and args["--warmup"] >= 3 and args["--steps"] >= 1
