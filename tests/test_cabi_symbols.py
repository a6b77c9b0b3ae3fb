"""The C-ABI shared library loads (no GPU needed) and exports every entry point include/vstar_b200.h declares; the
ctypes table in vstar_b200/_lib.py covers exactly those symbols.  No compute calls here."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared():
    src = open(os.path.join(ROOT, "include", "vstar_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(vsb_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from vstar_b200 import _lib, build
    build.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    names = declared()
    assert len(names) >= 30
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/vstar_b200.h but not exported"
    table = set(_lib.SIGNATURES) | {"vsb_last_error", "vsb_version"}
    assert table == set(names), (sorted(table - set(names)), sorted(set(names) - table))
    loaded = _lib.load()
    assert loaded.vsb_version() >= 100 and isinstance(loaded.vsb_last_error(), bytes)


def test_ops_refuse_cpu_tensors_without_fallback():
    import pytest
    import torch
    from vstar_b200 import ops
    from vstar_b200._lib import VsbError
    with pytest.raises(VsbError):
        ops.gemm(torch.zeros(8, 8, dtype=torch.bfloat16), torch.zeros(8, 8, dtype=torch.bfloat16))
    with pytest.raises(VsbError):
        ops.layernorm(torch.zeros(8, 8, dtype=torch.bfloat16), torch.ones(8, dtype=torch.bfloat16), torch.zeros(8, dtype=torch.bfloat16), 1e-5)


def test_ctypes_table_matches_the_header_prototypes():
    """argument count and kind (pointer / integer / float) of every prototype in include/vstar_b200.h against the ctypes
    argtypes the Python host uses - a mismatch would corrupt the call silently"""
    from vstar_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vstar_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    protos = dict(re.findall(r"\bint\s+(vsb_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", src, flags=re.S))
    assert set(_lib.SIGNATURES) <= set(protos), sorted(set(_lib.SIGNATURES) - set(protos))

    def kind_c(param):
        param = " ".join(param.split())
        if param in ("void", ""):
            return None
        if "*" in param:
            return "p"
        if param.startswith("float") or param.startswith("double"):
            return "f"
        assert re.match(r"(const )?(int|long long)\b", param), param
        return "i"

    def kind_py(t):
        if t in (ctypes.c_float, ctypes.c_double):
            return "f"
        if t in (ctypes.c_int, ctypes.c_longlong):
            return "i"
        return "p"                                  # c_void_p, POINTER(...)

    for name, argtypes in _lib.SIGNATURES.items():
        want = [k for k in (kind_c(p) for p in protos[name].split(",")) if k is not None]
        got = [kind_py(t) for t in argtypes]
        assert got == want, (name, got, want)
        # widths of the integer arguments as well
        c_ints = [("long long" in " ".join(p.split())) for p in protos[name].split(",") if kind_c(p) == "i"]
        py_ints = [t is ctypes.c_longlong for t in argtypes if kind_py(t) == "i"]
        assert c_ints == py_ints, (name, c_ints, py_ints)


def test_layer_struct_matches_the_header():
    """member names of vsb_llama_layer_t in include/vstar_b200.h, in order, against the ctypes struct the layer table is built
    from - the runner reads the table by field offset"""
    from vstar_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vstar_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    body = re.search(r"typedef struct \{([^}]*)\} vsb_llama_layer_t;", src).group(1)
    members = re.findall(r"const void\* (\w+);", body)
    assert len(members) == len(body.split(";")) - 1, body
    assert members == [name for name, _ in _lib.LlamaLayer._fields_]
    assert all(t is ctypes.c_void_p for _, t in _lib.LlamaLayer._fields_)
