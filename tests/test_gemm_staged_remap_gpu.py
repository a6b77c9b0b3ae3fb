"""The staged epilogue of the wgmma tile GEMM writes T output through per-warp shared-memory slots of 16 rows x 32 columns, each
slot row leaving as one bulk copy to its (possibly remapped) output row, clipped at M and at the output width.  Each case runs
the same problem twice into a sentinel-filled C: once staged, once on the direct path that stores from the accumulator
registers, and checks
  * both outputs (the whole buffer, sentinels included) are equal bit for bit;
  * every element outside the written rows and columns still holds the sentinel, every element inside is finite.
Cases: row remaps (KV-cache layout: group_offset > 0, gaps between groups) with 1 to 283 rows per group, M a multiple of the
group size or not; partial last m-tiles; output widths that end in a partial 32-column chunk; SwiGLU; in-place residual; the
fused QKV + RoPE projection into a KV-cache-shaped buffer; bf16 and f16.
The direct path is reached by placing C 8 bytes past a 16-byte boundary (small shapes) or, on shapes of at least 512 x 512 x 1024,
by the streaming-store switch (vsb_gemm_set_l2_hints bit 2), which keeps C 16-byte aligned: vsb_gemm_qkv_rope_* requires that.
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
DTYPES = [torch.bfloat16, torch.float16]
SENTINEL = 0x7FA5                      # a NaN in both bf16 and f16
OFF, PAD = 7, 3                        # row remap: group_offset, and group_stride = rows_per_group + PAD


def _cpu(shape, seed, dtype, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _rows(M, rpg, stride, off):
    """output row of every logical row m, and the number of rows the buffer needs (two spare rows after the last)"""
    m = torch.arange(M)
    r = m if rpg <= 0 else (m // rpg) * stride + off + m % rpg
    return r, int(r.max()) + 3


def _buffer(dt, rows, ldc, shift):
    """a C of rows x ldc filled with the sentinel, `shift` elements past a 16-byte boundary"""
    buf = torch.full((rows * ldc + 8,), SENTINEL, dtype=torch.int16, device="cuda").view(dt)
    assert buf.data_ptr() % 16 == 0
    return buf[shift:shift + rows * ldc].view(rows, ldc)


def _check(staged, direct, written, n_out):
    s16, d16 = staged.view(torch.int16), direct.view(torch.int16)
    assert torch.equal(s16, d16)
    mask = torch.zeros(staged.shape, dtype=torch.bool, device=staged.device)
    mask[written.to(staged.device), :n_out] = True
    assert (s16[~mask] == SENTINEL).all()
    assert torch.isfinite(staged[mask].float()).all()


def gemm(dt, M, N, K, epi, res, rpg, ldc, shift):
    """C = epi(A W^T + bias) (+ C in place), rows remapped by (rpg, rpg + PAD, OFF) unless rpg <= 0"""
    from vstar_b200 import _lib
    n_out = N // 2 if epi == EPI_SWIGLU else N
    stride = rpg + PAD if rpg > 0 else 0
    written, rows = _rows(M, rpg, stride, OFF)
    a = _cpu((M, K), 1, dt)
    w = _cpu((N, K), 2, dt, scale=K ** -0.5)
    bias = _cpu((N,), 3, dt, scale=0.5)
    out = _buffer(dt, rows, ldc, shift)
    if res:
        out[written.cuda(), :n_out] = _cpu((M, n_out), 4, dt)
    _lib.call("vsb_gemm_" + SFX[dt], a.data_ptr(), K, w.data_ptr(), K, out.data_ptr(), ldc, M, N, K, bias.data_ptr(),
              out.data_ptr() if res else None, ldc if res else 0, epi, 0, max(rpg, 0), stride, OFF if rpg > 0 else 0, _stream())
    torch.cuda.synchronize()
    return out.clone(), written, n_out


# (rows per group (0: no remap), M): partial last 128-row tiles, M a multiple of the group size or ending in a partial group
REMAPS = [(0, 210), (1, 200), (5, 205), (15, 210), (16, 208), (17, 221), (283, 566), (17, 215), (283, 500)]
# name -> N, epilogue, in-place residual; N = 520 and SwiGLU's 264 output columns end in a partial 32-column chunk
EPIS = {"bias": (520, EPI_NONE, False), "residual": (520, EPI_NONE, True), "swiglu": (528, EPI_SWIGLU, False)}


@pytest.mark.parametrize("dt", DTYPES, ids=["bf16", "f16"])
@pytest.mark.parametrize("epi", list(EPIS))
@pytest.mark.parametrize("rpg,M", REMAPS, ids=[f"rpg{r}-M{m}" for r, m in REMAPS])
@pytest.mark.parametrize("bn,ctas", [(64, 0), (128, 3), (256, 0)])
def test_staged_equals_direct(bn, ctas, rpg, M, epi, dt):
    from vstar_b200 import _lib
    N, e, res = EPIS[epi]
    ldc = (N // 2 if e == EPI_SWIGLU else N) + 8          # columns past the output width must stay untouched
    _lib.call("vsb_gemm_set_tuning", bn, ctas)
    try:
        staged, written, n_out = gemm(dt, M, N, 200, e, res, rpg, ldc, 0)
        direct, _, _ = gemm(dt, M, N, 200, e, res, rpg, ldc, 4)     # 8 bytes past a 16-byte boundary: direct
    finally:
        _lib.call("vsb_gemm_set_tuning", 0, 0)
    _check(staged, direct, written, n_out)


@pytest.mark.parametrize("dt", DTYPES, ids=["bf16", "f16"])
def test_single_group_with_offset(dt):
    """rows_per_group >= M: one group of rows starting at row group_offset"""
    from vstar_b200 import _lib
    M, N, K, ldc = 150, 264, 128, 272
    written = torch.arange(M) + OFF
    out = []
    for shift in (0, 4):
        a, w = _cpu((M, K), 1, dt), _cpu((N, K), 2, dt, scale=K ** -0.5)
        c = _buffer(dt, M + OFF + 2, ldc, shift)
        _lib.call("vsb_gemm_" + SFX[dt], a.data_ptr(), K, w.data_ptr(), K, c.data_ptr(), ldc, M, N, K, None, None, 0, EPI_NONE, 0,
                  M + 5, 0, OFF, _stream())
        torch.cuda.synchronize()
        out.append(c.clone())
    _check(out[0], out[1], written, N)


def _streaming(fn):
    from vstar_b200 import _lib
    staged = fn()
    _lib.call("vsb_gemm_set_l2_hints", 4)
    try:
        direct = fn()
    finally:
        _lib.call("vsb_gemm_set_l2_hints", 0)
    return staged, direct


@pytest.mark.parametrize("dt", DTYPES, ids=["bf16", "f16"])
def test_large_remap_residual_equals_streaming(dt):
    M, N, K, rpg = 17 * 32, 520, 1024, 17
    staged, direct = _streaming(lambda: gemm(dt, M, N, K, EPI_NONE, True, rpg, N + 8, 0))
    _check(staged[0], direct[0], staged[1], N)


@pytest.mark.parametrize("dt", DTYPES, ids=["bf16", "f16"])
def test_qkv_rope_kv_cache_equals_streaming(dt):
    """fused QKV + RoPE into a [B, T_max, 3d] KV-cache-shaped buffer at rows [past, past + T) of each sequence"""
    from vstar_b200 import _lib
    B, T, TMAX, PAST, d, K = 2, 283, 384, 37, 256, 1024
    M, N = B * T, 3 * d
    a = _cpu((M, K), 1, dt)
    w = _cpu((N, K), 2, dt, scale=K ** -0.5)
    sq_in = (torch.rand(K // 32, M, generator=torch.Generator().manual_seed(5)) + 0.5).mul(32.0).cuda()
    pos = torch.arange(2048, dtype=torch.float32)[:, None]
    ang = pos / (10000.0 ** (torch.arange(0, 128, 2, dtype=torch.float32) / 128))
    cos, sin = ang.cos().to(dt).cuda().contiguous(), ang.sin().to(dt).cuda().contiguous()
    written = (torch.arange(M) // T) * TMAX + PAST + torch.arange(M) % T

    def run():
        c = _buffer(dt, B * TMAX, N, 0)
        _lib.call("vsb_gemm_qkv_rope_" + SFX[dt], a.data_ptr(), K, w.data_ptr(), K, c.data_ptr(), N, M, N, K, T, TMAX, PAST,
                  sq_in.data_ptr(), K // 32, 1e-6, M, cos.data_ptr(), sin.data_ptr(), None, T, PAST, 128, _stream())
        torch.cuda.synchronize()
        return c.clone()

    staged, direct = _streaming(run)
    _check(staged, direct, written, N)
