"""Edge cases of the wgmma tile GEMM's epilogue, bit for bit.

Every forced tile width x {no epilogue, bias + GELU, in-place residual, bias + SwiGLU, fp32 output with in-place residual, folded
RMSNorm in, folded RMSNorm out with in-place residual, fused RoPE, odd ldc}, at M = 210 and N not a multiple of the tile (partial
tiles in both directions), in bf16 and f16, with one CTA per tile and with 3 CTAs looping over every tile.  Each case checks:
  * the call writing through a row remap whose groups straddle tiles (70 rows per group at a stride of 96, the KV-cache layout)
    equals the same call with a contiguous, unremapped output, bit for bit;
  * the contiguous output (and the row statistics, where written) hashes to the sha256 digest stored in
    tests/golden/gemm_epilogue_digests.json, generated with an earlier build of the library: the epilogue's arithmetic is pinned.

Inputs are seeded on the CPU and copied to the device.  Regenerate the digests (only when the epilogue's results are meant to
change) with
    python tests/test_gemm_epilogue_gpu.py [--lib path/to/libvstar_b200.so] [--out digests.json]
"""
import argparse
import hashlib
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

DIGESTS = os.path.join(ROOT, "tests", "golden", "gemm_epilogue_digests.json")
M, K, TN, TMAX, OFF = 210, 200, 70, 96, 13          # row remap: m -> (m // TN) * TMAX + OFF + m % TN
EPI_NONE, EPI_GELU, EPI_SWIGLU = 0, 2, 4
SFX = {torch.bfloat16: "bf16", torch.float16: "f16"}

# name: N, epilogue, bias, residual (added in place), fp32 output, rowsq_in chunks, rowsq_out, fused RoPE, odd ldc
CASES = {
    "none": dict(N=520),
    "bias_gelu": dict(N=520, epi=EPI_GELU, bias=True),
    "residual": dict(N=520, res=True),
    "swiglu": dict(N=528, epi=EPI_SWIGLU, bias=True),
    "fp32_out": dict(N=520, bias=True, res=True, fp32=True),
    "fold_in": dict(N=520, sq_in=5),
    "fold_out": dict(N=512, res=True, sq_out=True),
    "rope": dict(N=768, sq_in=3, rope=True),
    "odd_ldc": dict(N=520, bias=True, res=True, odd=True),
}


def _cpu(shape, seed, dtype, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def _remap(m):
    return (m // TN) * TMAX + OFF + m % TN


def run_case(name, dt, remapped):
    """-> list of output tensors of the case, read back as the rows of the logical [M, n_out] result"""
    from vstar_b200 import _lib
    c = CASES[name]
    N = c["N"]
    epi = c.get("epi", EPI_NONE)
    n_out = N // 2 if epi == EPI_SWIGLU else N
    odt = torch.float32 if c.get("fp32") else dt
    a = _cpu((M, K), 1, dt)
    w = _cpu((N, K), 2, dt, scale=K ** -0.5)
    bias = _cpu((N,), 3, dt, scale=0.5) if c.get("bias") else None
    res = _cpu((M, n_out), 4, odt) if c.get("res") else None
    idx = torch.tensor([_remap(m) for m in range(M)], device="cuda") if remapped else torch.arange(M, device="cuda")
    rows = (M // TN + 1) * TMAX if remapped else M
    sq_in = None
    if c.get("sq_in"):
        # rowsq_in and rowsq_out share the leading dimension sq_ld = rows (rowsq_out is indexed by the remapped row)
        g = torch.Generator(device="cpu").manual_seed(5)
        sq_in = torch.zeros(c["sq_in"], rows, device="cuda")
        sq_in[:, :M] = (torch.rand(c["sq_in"], M, generator=g) * K / c["sq_in"] + 1.0).cuda()
    ldc = n_out + 1 if (c.get("odd") and remapped) else n_out
    buf = torch.zeros(rows * ldc, dtype=odt, device="cuda")
    out = buf.view(rows, ldc)
    if res is not None:
        out[idx, :n_out] = res                            # the residual is added in place: residual == C
    sq_out = torch.full((N // 32, rows), -1.0, device="cuda") if c.get("sq_out") else None
    rpg, gs, go = (TN, TMAX, OFF) if remapped else (0, 0, 0)
    p = lambda t: 0 if t is None else t.data_ptr()  # noqa: E731
    stream = torch.cuda.current_stream().cuda_stream
    sfx = SFX[dt]
    if c.get("rope"):
        pos = torch.arange(512, dtype=torch.float32)[:, None] * (10000.0 ** (-torch.arange(0, 64, dtype=torch.float32) / 64))
        cos, sin = pos.cos().to(dt).cuda(), pos.sin().to(dt).cuda()
        _lib.call("vsb_gemm_qkv_rope_" + sfx, a.data_ptr(), K, w.data_ptr(), K, out.data_ptr(), ldc, M, N, K, rpg, gs, go, p(sq_in),
                  sq_in.shape[0], 1e-6, rows, cos.data_ptr(), sin.data_ptr(), None, TN, 7, 128, stream)
    elif sq_in is not None or sq_out is not None:
        _lib.call("vsb_gemm_rowscale_" + sfx, a.data_ptr(), K, w.data_ptr(), K, out.data_ptr(), ldc, M, N, K, p(bias),
                  p(out) if res is not None else None, ldc if res is not None else 0, epi, rpg, gs, go, p(sq_in),
                  sq_in.shape[0] if sq_in is not None else 0, 1e-6, p(sq_out), rows, stream)
    else:
        _lib.call("vsb_gemm_" + sfx, a.data_ptr(), K, w.data_ptr(), K, out.data_ptr(), ldc, M, N, K, p(bias),
                  p(out) if res is not None else None, ldc if res is not None else 0, epi, 1 if odt == torch.float32 else 0, rpg, gs, go,
                  stream)
    torch.cuda.synchronize()
    outs = [out[idx, :n_out].contiguous()]
    if sq_out is not None:
        outs.append(sq_out[:, idx].contiguous())
    return outs


def digest(t):
    t = t.contiguous().cpu()
    return hashlib.sha256(t.view({2: torch.int16, 4: torch.int32}[t.element_size()]).numpy().tobytes()).hexdigest()


def case_digests(name, dt, bn, max_ctas=0):
    from vstar_b200 import _lib
    _lib.call("vsb_gemm_set_tuning", bn, max_ctas)
    try:
        plain = run_case(name, dt, remapped=False)
        remapped = run_case(name, dt, remapped=True)
    finally:
        _lib.call("vsb_gemm_set_tuning", 0, 0)
    return plain, remapped


def key(name, dt, bn):
    return f"{name}.{SFX[dt]}.bn{bn}"


@pytest.fixture(scope="module")
def golden():
    with open(DIGESTS) as f:
        return json.load(f)


@pytest.mark.parametrize("max_ctas", [0, 3])
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
@pytest.mark.parametrize("bn", [32, 64, 128, 256])
@pytest.mark.parametrize("name", list(CASES))
def test_gemm_epilogue_bits(golden, name, bn, dt, max_ctas):
    plain, remapped = case_digests(name, dt, bn, max_ctas)
    for x, y in zip(plain, remapped):
        assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), f"{name}: remapped output differs from the contiguous one"
    assert torch.isfinite(plain[0].float()).all()
    assert [digest(x) for x in plain] == golden[key(name, dt, bn)], f"{key(name, dt, bn)}: output bits changed"


if __name__ == "__main__":
    ap = argparse.ArgumentParser(description="regenerate " + os.path.relpath(DIGESTS, ROOT))
    ap.add_argument("--lib", default=None, help="libvstar_b200.so to load instead of the in-tree build")
    ap.add_argument("--out", default=DIGESTS)
    args = ap.parse_args()
    from vstar_b200 import _lib
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    res = {}
    for name in CASES:
        for dt in SFX:
            for bn in (32, 64, 128, 256):
                plain, remapped = case_digests(name, dt, bn)
                assert all(torch.equal(x.view(torch.uint8), y.view(torch.uint8)) for x, y in zip(plain, remapped)), key(name, dt, bn)
                res[key(name, dt, bn)] = [digest(x) for x in plain]
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
    print(f"{len(res)} digests -> {args.out}")
