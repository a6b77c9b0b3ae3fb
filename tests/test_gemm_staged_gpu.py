"""The wgmma tile GEMM writes T output either through shared memory with bulk copies (staged) or straight from the accumulator
registers (direct), chosen from what the launch allows.  The boundaries of that choice that tests/test_gemm_epilogue_gpu.py does
not reach, each checked bit for bit against the staged path on the same problem:
  * C 8-byte but not 16-byte aligned, with ldc % 8 == 0: direct;
  * streaming output stores (vsb_gemm_set_l2_hints bit 2, large GEMMs only): direct.
"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

EPI_NONE, EPI_SWIGLU = 0, 4
SFX = {torch.bfloat16: "bf16", torch.float16: "f16"}


def _cpu(shape, seed, dtype, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def gemm(dt, M, N, K, epi, shift):
    """C = epi(A W^T + bias) (+ C in place unless SwiGLU), written at element offset `shift` of a 16-byte aligned buffer"""
    from vstar_b200 import _lib
    n_out = N // 2 if epi == EPI_SWIGLU else N
    a = _cpu((M, K), 1, dt)
    w = _cpu((N, K), 2, dt, scale=K ** -0.5)
    bias = _cpu((N,), 3, dt, scale=0.5)
    buf = torch.zeros(M * n_out + 8, dtype=dt, device="cuda")
    assert buf.data_ptr() % 16 == 0
    out = buf[shift:shift + M * n_out].view(M, n_out)
    res = epi != EPI_SWIGLU
    if res:
        out.copy_(_cpu((M, n_out), 4, dt))
    _lib.call("vsb_gemm_" + SFX[dt], a.data_ptr(), K, w.data_ptr(), K, out.data_ptr(), n_out, M, N, K, bias.data_ptr(),
              out.data_ptr() if res else None, n_out if res else 0, epi, 0, 0, 0, 0, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out.clone()


def _same(x, y):
    return torch.equal(x.view(torch.int16), y.view(torch.int16))


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
@pytest.mark.parametrize("epi", [EPI_NONE, EPI_SWIGLU], ids=["residual", "swiglu"])
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_c_8_byte_aligned_direct_equals_staged(bn, epi, dt):
    from vstar_b200 import _lib
    _lib.call("vsb_gemm_set_tuning", bn, 0)
    try:
        staged = gemm(dt, 210, 528, 200, epi, 0)
        direct = gemm(dt, 210, 528, 200, epi, 4)      # 8 bytes past a 16-byte boundary; ldc = 528 or 264, both % 8 == 0
    finally:
        _lib.call("vsb_gemm_set_tuning", 0, 0)
    assert torch.isfinite(staged.float()).all()
    assert _same(staged, direct)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
def test_streaming_stores_direct_equals_staged(dt):
    from vstar_b200 import _lib
    staged = gemm(dt, 640, 1024, 1024, EPI_NONE, 0)
    _lib.call("vsb_gemm_set_l2_hints", 4)
    try:
        direct = gemm(dt, 640, 1024, 1024, EPI_NONE, 0)
    finally:
        _lib.call("vsb_gemm_set_l2_hints", 0)
    assert _same(staged, direct)
