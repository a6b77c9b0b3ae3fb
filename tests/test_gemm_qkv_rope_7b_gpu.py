"""vsb_llama_layers runs the QKV projection and RoPE as two kernels by default and as one GEMM with a RoPE epilogue when
vsb_llama_set_fuse_rope(1) is set: both must leave the same bits in the KV cache.  At the Llama-7B width (d = 4096, 32 heads of
128, K = 4096) each case compares the fused QKV + RoPE projection (vsb_gemm_qkv_rope_*) bit for bit with the same GEMM without
RoPE (vsb_gemm_rowscale_*, folded RMSNorm in) followed by vsb_rope_*, both writing into a sentinel-filled [B, T_max, 3d]
KV-cache-shaped buffer at rows [past, past + T) of each sequence:
  * the two buffers are equal bit for bit, sentinels included;
  * every row outside the written ones still holds the sentinel, every written element is finite.
Cases: 64 crops of 283 rows (a partial last 128-row tile) with positions pos0 + m % T or from a per-row table; 32 crops of 5
rows; 2 crops on 3 CTAs, so the shared-memory ring and the row-scale slots wrap their phases across many tiles per CTA; bf16
and f16.
"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

SFX = {torch.bfloat16: "bf16", torch.float16: "f16"}
SENTINEL = 0x7FA5                      # a NaN in both bf16 and f16
D, H, HD, TMAX, PAST, MAXPOS = 4096, 32, 128, 384, 37, 2048

# name -> (crops, rows per crop, per-row positions table, max CTAs (0: one per SM))
CASES = {"b64-pos0": (64, 283, False, 0), "b64-positions": (64, 283, True, 0), "b32x5": (32, 5, False, 0), "b2-ctas3": (2, 283, False, 3)}


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _randn(shape, seed, dtype, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(dtype)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16], ids=["bf16", "f16"])
@pytest.mark.parametrize("case", list(CASES))
def test_qkv_rope_equals_gemm_then_rope(case, dt):
    from vstar_b200 import _lib
    B, T, table, ctas = CASES[case]
    M, N, K = B * T, 3 * D, D
    sfx = SFX[dt]
    a = _randn((M, K), 1, dt)
    w = _randn((N, K), 2, dt, scale=K ** -0.5)
    g = torch.Generator(device="cuda").manual_seed(3)
    sq_in = (torch.rand(K // 32, M, generator=g, device="cuda") + 0.5) * 32.0     # folded RMSNorm: 128 partial sums per row
    pos = torch.arange(MAXPOS, dtype=torch.float32)[:, None]
    ang = pos / (10000.0 ** (torch.arange(0, HD, 2, dtype=torch.float32) / HD))
    cos, sin = ang.cos().to(dt).cuda().contiguous(), ang.sin().to(dt).cuda().contiguous()
    positions = torch.randint(0, MAXPOS, (M,), generator=g, device="cuda", dtype=torch.int32) if table else None
    pp = positions.data_ptr() if table else None
    written = ((torch.arange(M) // T) * TMAX + PAST + torch.arange(M) % T).cuda()

    def cache():
        return torch.full((B * TMAX, N), SENTINEL, dtype=torch.int16, device="cuda").view(dt)

    fused, ref = cache(), cache()
    _lib.call("vsb_gemm_set_tuning", 0, ctas)
    try:
        _lib.call("vsb_gemm_qkv_rope_" + sfx, a.data_ptr(), K, w.data_ptr(), K, fused.data_ptr(), N, M, N, K, T, TMAX, PAST,
                  sq_in.data_ptr(), K // 32, 1e-6, M, cos.data_ptr(), sin.data_ptr(), pp, T, PAST, HD, _stream())
        _lib.call("vsb_gemm_rowscale_" + sfx, a.data_ptr(), K, w.data_ptr(), K, ref.data_ptr(), N, M, N, K, None, None, 0, 0, T, TMAX,
                  PAST, sq_in.data_ptr(), K // 32, 1e-6, None, M, _stream())
        _lib.call("vsb_rope_" + sfx, ref.data_ptr(), N, M, T, H, HD, PAST, cos.data_ptr(), sin.data_ptr(), pp, TMAX, PAST, _stream())
        torch.cuda.synchronize()
    finally:
        _lib.call("vsb_gemm_set_tuning", 0, 0)
    f16, r16 = fused.view(torch.int16), ref.view(torch.int16)
    assert torch.equal(f16, r16)
    mask = torch.zeros(B * TMAX, dtype=torch.bool, device="cuda")
    mask[written] = True
    assert (f16[~mask] == SENTINEL).all()
    assert torch.isfinite(fused[mask].float()).all()
