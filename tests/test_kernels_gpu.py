"""Per-kernel parity on a real H100: every C-ABI entry point against the same op in plain PyTorch
(fp32 math on the same bf16-rounded inputs).  Tolerances are written per test."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BF = torch.bfloat16


@pytest.fixture(scope="module")
def ops():
    from vstar_b200 import ops as o
    return o


def rnd(*shape, scale=1.0, seed=0, dtype=BF):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def rel_err(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


GEMM_SHAPES = [
    (128, 128, 64), (128, 256, 128), (256, 512, 256), (1, 128, 64), (5, 4, 768), (257, 1024, 1024),
    (300, 514, 768), (640, 11008, 512), (2304, 768, 768), (320, 4096, 4096), (77, 200, 592), (128, 64, 2304),
    (1280, 8192, 1024), (16, 4096, 2048), (5, 4096, 1024), (100, 1056, 512),
]


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_plain(ops, M, N, K):
    a, w = rnd(M, K, seed=1), rnd(N, K, scale=1 / math.sqrt(K), seed=2)
    out = ops.gemm(a, w)
    ref = a.float() @ w.float().t()
    torch.cuda.synchronize()
    assert out.shape == (M, N)
    # bf16 output rounding: rel 2^-8 of the value + fp32 accumulation noise
    assert torch.allclose(out.float(), ref, rtol=1e-2, atol=2e-2), rel_err(out, ref)


@pytest.mark.parametrize("bn", [32, 64, 128, 256])
def test_gemm_forced_tile(ops, bn):
    from vstar_b200 import _lib
    M, N, K = 384, 768, 320
    a, w = rnd(M, K, seed=3), rnd(N, K, scale=1 / math.sqrt(K), seed=4)
    _lib.call("vsb_gemm_set_tuning", bn, 0)
    try:
        out = ops.gemm(a, w, out_dtype=torch.float32)
    finally:
        _lib.call("vsb_gemm_set_tuning", 0, 0)
    ref = a.float() @ w.float().t()
    assert torch.allclose(out, ref, rtol=1e-4, atol=1e-3), rel_err(out, ref)


@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (512, 512, 256), (2560, 4096, 512), (300, 514, 768), (1000, 1280, 320),
                                   (129, 257, 128), (2048, 11008, 256), (4096, 768, 768)])
def test_gemm_wide_tile(ops, M, N, K):
    """128 x 256 tiles (the widest wgmma tile) with bias / activation / residual on even / ragged shapes"""
    from vstar_b200 import _lib
    a, w, b, r = rnd(M, K, seed=31), rnd(N, K, scale=1 / math.sqrt(K), seed=32), rnd(N, seed=33), rnd(M, N, seed=34)
    _lib.call("vsb_gemm_set_tuning", 256, 0)
    try:
        out = ops.gemm(a, w, out_dtype=torch.float32)
        out2 = ops.gemm(a, w, bias=b, residual=r, epilogue=ops.EPI_QUICK_GELU)
    finally:
        _lib.call("vsb_gemm_set_tuning", 0, 0)
    ref = a.float() @ w.float().t()
    assert torch.allclose(out, ref, rtol=1e-4, atol=1e-3), rel_err(out, ref)
    y = ref + b.float()
    ref2 = y * torch.sigmoid(1.702 * y) + r.float()
    assert torch.allclose(out2.float(), ref2, rtol=1e-2, atol=3e-2), rel_err(out2, ref2)


def test_gemm_wide_tile_persistent_few_ctas(ops):
    from vstar_b200 import _lib
    M, N, K = 1536, 2048, 448
    a, w = rnd(M, K, seed=35), rnd(N, K, scale=1 / math.sqrt(K), seed=36)
    _lib.call("vsb_gemm_set_tuning", 256, 3)          # 3 CTAs, 96 tiles -> 32 tiles each: smem ring phases across tiles
    try:
        out = ops.gemm(a, w, out_dtype=torch.float32)
    finally:
        _lib.call("vsb_gemm_set_tuning", 0, 0)
    ref = a.float() @ w.float().t()
    assert torch.allclose(out, ref, rtol=1e-4, atol=1e-3), rel_err(out, ref)


@pytest.mark.parametrize("group_m", [1, 3, 8, 64])
def test_gemm_tile_rasterisation(ops, group_m):
    from vstar_b200 import _lib
    M, N, K = 1500, 1300, 192
    a, w = rnd(M, K, seed=37), rnd(N, K, scale=1 / math.sqrt(K), seed=38)
    _lib.call("vsb_gemm_set_group_m", group_m)
    try:
        out = ops.gemm(a, w, out_dtype=torch.float32)
        _lib.call("vsb_gemm_set_tuning", 256, 0)
        out2 = ops.gemm(a, w, out_dtype=torch.float32)
    finally:
        _lib.call("vsb_gemm_set_group_m", 0)
        _lib.call("vsb_gemm_set_tuning", 0, 0)
    ref = a.float() @ w.float().t()
    assert torch.allclose(out, ref, rtol=1e-4, atol=1e-3) and torch.allclose(out2, ref, rtol=1e-4, atol=1e-3)


def test_gemm_persistent_many_tiles(ops):
    """few CTAs, many tiles per CTA: exercises the smem ring phases across tiles"""
    from vstar_b200 import _lib
    M, N, K = 1024, 1536, 448
    a, w = rnd(M, K, seed=5), rnd(N, K, scale=1 / math.sqrt(K), seed=6)
    _lib.call("vsb_gemm_set_tuning", 128, 3)
    try:
        out = ops.gemm(a, w, out_dtype=torch.float32)
    finally:
        _lib.call("vsb_gemm_set_tuning", 0, 0)
    ref = a.float() @ w.float().t()
    assert torch.allclose(out, ref, rtol=1e-4, atol=1e-3), rel_err(out, ref)


@pytest.mark.parametrize("epi", ["none", "quick_gelu", "gelu", "relu"])
def test_gemm_bias_act_residual(ops, epi):
    M, N, K = 515, 1000, 256
    a, w, b, r = rnd(M, K, seed=7), rnd(N, K, scale=1 / math.sqrt(K), seed=8), rnd(N, seed=9), rnd(M, N, seed=10)
    code = dict(none=ops.EPI_NONE, quick_gelu=ops.EPI_QUICK_GELU, gelu=ops.EPI_GELU, relu=ops.EPI_RELU)[epi]
    out = ops.gemm(a, w, bias=b, residual=r, epilogue=code)
    y = a.float() @ w.float().t() + b.float()
    y = dict(none=lambda t: t, quick_gelu=lambda t: t * torch.sigmoid(1.702 * t), gelu=F.gelu, relu=F.relu)[epi](y)
    ref = y + r.float()
    assert torch.allclose(out.float(), ref, rtol=1e-2, atol=3e-2), rel_err(out, ref)


def test_gemm_swiglu(ops):
    M, I, K = 200, 704, 256
    a = rnd(M, K, seed=11)
    gate, up = rnd(I, K, scale=1 / math.sqrt(K), seed=12), rnd(I, K, scale=1 / math.sqrt(K), seed=13)
    w = torch.stack([gate, up], dim=1).reshape(2 * I, K).contiguous()     # interleaved rows
    out = ops.gemm(a, w, epilogue=ops.EPI_SWIGLU)
    ref = F.silu(a.float() @ gate.float().t()) * (a.float() @ up.float().t())
    assert out.shape == (M, I)
    assert torch.allclose(out.float(), ref, rtol=1e-2, atol=2e-2), rel_err(out, ref)


def test_gemm_row_remap_and_strided(ops):
    """scatter 256-row groups into a [B, T, d] buffer at offset p (the mm_projector -> LLM input path)"""
    B, G, K, N, T, p0 = 3, 256, 128, 512, 300, 20
    a, w, b = rnd(B * G, K, seed=14), rnd(N, K, scale=1 / math.sqrt(K), seed=15), rnd(N, seed=16)
    buf = torch.zeros(B * T, N, dtype=BF, device="cuda")
    ops.gemm(a, w, out=buf, bias=b, rows_per_group=G, group_stride=T, group_offset=p0)
    ref = (a.float() @ w.float().t() + b.float()).view(B, G, N)
    got = buf.view(B, T, N)
    assert torch.allclose(got[:, p0:p0 + G].float(), ref, rtol=1e-2, atol=2e-2)
    assert float(got[:, :p0].abs().max()) == 0 and float(got[:, p0 + G:].abs().max()) == 0
    # strided A (a column slice of a wider matrix) and strided output
    wide = rnd(100, 3 * K, seed=17)
    o2 = torch.zeros(100, 2 * N, dtype=BF, device="cuda")
    ops.gemm(wide[:, K:2 * K], w, out=o2[:, N:])
    assert torch.allclose(o2[:, N:].float(), wide[:, K:2 * K].float() @ w.float().t(), rtol=1e-2, atol=2e-2)
    assert float(o2[:, :N].abs().max()) == 0


@pytest.mark.parametrize("D,causal,Sq,Sk", [(64, False, 1, 2305), (64, True, 4, 130), (128, False, 2, 700)])
def test_attn_decode_kernel_shapes(ops, D, causal, Sq, Sk):
    from vstar_b200 import _lib
    B, H = 2, 3
    q, k, v = rnd(B * Sq, H * D, seed=44), rnd(B * Sk, H * D, seed=45), rnd(B * Sk, H * D, seed=46)
    out = torch.empty(B * Sq, H * D, dtype=BF, device="cuda")
    _lib.call("vsb_attn_set_impl", 4)
    try:
        ops.flash_attn(q, k, v, out, B, H, Sq, Sk, D, causal, D ** -0.5, Sq * H * D, H * D, Sk * H * D, H * D, Sk * H * D, H * D, Sq * H * D, H * D)
        torch.cuda.synchronize()
    finally:
        _lib.call("vsb_attn_set_impl", 0)
    qf, kf, vf = [t.view(B, -1, H, D).transpose(1, 2).float() for t in (q, k, v)]
    att = qf @ kf.transpose(-1, -2) * D ** -0.5
    if causal:
        att = att.masked_fill(~torch.ones(Sq, Sk, device="cuda").tril(Sk - Sq).bool(), float("-inf"))
    ref = (torch.softmax(att, -1) @ vf).transpose(1, 2).reshape(B * Sq, H * D)
    assert torch.allclose(out.float(), ref, rtol=2e-2, atol=2e-2), rel_err(out, ref)


@pytest.mark.parametrize("M,N,K", [(1, 4096, 4096), (1, 1001, 1000), (2, 514, 768), (3, 77, 11008), (4, 2048, 264), (5, 333, 2048),
                                   (8, 12288, 1024), (7, 32004, 512), (9, 4096, 4096), (16, 1000, 1192), (13, 22016, 256)])
def test_gemm_skinny(ops, M, N, K):
    """decode-sized problems take the weight-streaming kernels of gemm_skinny.cu (CUDA-core FMA kernel for M <= 2, mma.sync
    kernel up to M = 16); both must agree with the fp32 reference AND with the wgmma tile kernel on every epilogue variant
    (same semantics behind vsb_gemm_bf16)"""
    from vstar_b200 import _lib
    a, w, b = rnd(M, K, seed=61), rnd(N, K, scale=1 / math.sqrt(K), seed=62), rnd(N, seed=63)
    r, r32 = rnd(M, N, seed=64), torch.randn(M, N, device="cuda")

    def run_all():
        o = [ops.gemm(a, w, out_dtype=torch.float32), ops.gemm(a, w, bias=b, residual=r, epilogue=ops.EPI_QUICK_GELU),
             ops.gemm(a, w, bias=b, epilogue=ops.EPI_GELU), ops.gemm(a, w, residual=r, epilogue=ops.EPI_RELU),
             ops.gemm(a, w, bias=b, residual=r32, out_dtype=torch.float32)]
        if N % 2 == 0:
            o.append(ops.gemm(a, w, epilogue=ops.EPI_SWIGLU))
        return o

    got = {}
    try:
        for variant in ([1] if M <= 8 else []) + [2, 64]:   # 1 = FMA kernel, 2 = mma.sync kernel, 64 = wgmma tile kernel
            _lib.call("vsb_gemm_set_tuning", variant, 0)     # forcing a skinny variant errors out if it cannot take the shape
            got[variant] = run_all()
    finally:
        _lib.call("vsb_gemm_set_tuning", 0, 0)
    auto = ops.gemm(a, w, out_dtype=torch.float32)
    assert torch.equal(auto, got[1 if M == 1 else (2 if (M <= 8 or N <= 8192) else 64)][0])      # production dispatch
    y = a.float() @ w.float().t()
    yb = y + b.float()
    refs = [y, yb * torch.sigmoid(1.702 * yb) + r.float(), F.gelu(yb), F.relu(y) + r.float(), yb + r32]
    if N % 2 == 0:
        refs.append(F.silu(y[:, 0::2]) * y[:, 1::2])
    for variant, outs in got.items():
        for i, (o_, ref) in enumerate(zip(outs, refs)):
            tol = dict(rtol=1e-4, atol=1e-3) if o_.dtype == torch.float32 else dict(rtol=1e-2, atol=3e-2)
            assert o_.shape == ref.shape and torch.allclose(o_.float(), ref, **tol), (variant, i, rel_err(o_, ref))


def test_gemm_skinny_row_remap_strided(ops):
    """decode writes its q|k|v row into the fused cache through the row remap; A / C are strided views"""
    B, K, N, T, p0 = 3, 512, 384, 40, 17
    a_wide, w, b = rnd(B, 2 * K, seed=65), rnd(N, K, scale=1 / math.sqrt(K), seed=66), rnd(N, seed=67)
    buf = torch.zeros(B * T, 2 * N, dtype=BF, device="cuda")
    from vstar_b200 import _lib
    ref = a_wide[:, K:].float() @ w.float().t() + b.float()
    for variant in (1, 2):
        buf.zero_()
        _lib.call("vsb_gemm_set_tuning", variant, 0)
        try:
            ops.gemm(a_wide[:, K:], w, out=buf[:, N:], bias=b, rows_per_group=1, group_stride=T, group_offset=p0)
        finally:
            _lib.call("vsb_gemm_set_tuning", 0, 0)
        got = buf.view(B, T, 2 * N)
        assert torch.allclose(got[:, p0, N:].float(), ref, rtol=1e-2, atol=2e-2)
        got[:, p0, N:] = 0
        assert float(got.abs().max()) == 0


def test_layernorm_rmsnorm(ops):
    for rows, cols in [(7, 64), (300, 768), (257, 1024), (33, 4096), (10, 256)]:
        x, w, b = rnd(rows, cols, seed=20), (1 + 0.1 * torch.randn(cols)).to(BF).cuda(), rnd(cols, scale=0.1, seed=21)
        y = ops.layernorm(x, w, b, 1e-5)
        ref = F.layer_norm(x.float(), (cols,), w.float(), b.float(), 1e-5)
        assert torch.allclose(y.float(), ref, rtol=1e-2, atol=1e-2), (rows, cols, rel_err(y, ref))
        y = ops.layernorm(x, w, b, 1e-6, act=ops.EPI_GELU)
        assert torch.allclose(y.float(), F.gelu(F.layer_norm(x.float(), (cols,), w.float(), b.float(), 1e-6)), rtol=1e-2, atol=1e-2)
        z = ops.rmsnorm(x, w, 1e-6)
        xf = x.float()
        refz = w.float() * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6)).to(BF).float()
        assert torch.allclose(z.float(), refz, rtol=1e-2, atol=1e-2), (rows, cols, rel_err(z, refz))


def _rope_tables(maxpos, D, theta=10000.0):
    inv = 1.0 / (theta ** (torch.arange(0, D, 2, dtype=torch.float32) / D))
    fr = torch.outer(torch.arange(maxpos, dtype=torch.float32), inv)
    return fr.cos().to(BF).cuda(), fr.sin().to(BF).cuda()


def test_rope_bit_exact(ops):
    B, T, H, D = 2, 37, 3, 128
    qkv = rnd(B * T, 3 * H * D, seed=30)
    cos_t, sin_t = _rope_tables(64, D)
    ref = qkv.clone().view(B, T, 3, H, D)
    cos = torch.cat([cos_t[:T], cos_t[:T]], -1)[None, :, None, :]
    sin = torch.cat([sin_t[:T], sin_t[:T]], -1)[None, :, None, :]

    def rot(x):
        return torch.cat([-x[..., D // 2:], x[..., :D // 2]], -1)

    for i in (0, 1):
        x = ref[:, :, i]
        ref[:, :, i] = (x * cos) + (rot(x) * sin)          # bf16 ops, like HF
    out = ops.rope_(qkv.clone(), T, H, D, cos_t, sin_t)
    assert torch.equal(out.view(B, T, 3, H, D), ref)
    # explicit positions (decode step)
    pos = torch.full((B * T,), 41, dtype=torch.int32, device="cuda")
    out2 = ops.rope_(qkv.clone(), T, H, D, cos_t, sin_t, positions=pos).view(B, T, 3, H, D)
    c41 = torch.cat([cos_t[41], cos_t[41]])
    s41 = torch.cat([sin_t[41], sin_t[41]])
    x = qkv.view(B, T, 3, H, D)[:, :, 0]
    assert torch.equal(out2[:, :, 0], (x * c41) + (rot(x) * s41))
    assert torch.equal(out2[:, :, 2], qkv.view(B, T, 3, H, D)[:, :, 2])


@pytest.mark.parametrize("impl", [1, 2, 3])
@pytest.mark.parametrize("B,H,S,D,causal", [(1, 2, 257, 64, False), (2, 3, 2305, 64, False), (2, 4, 320, 128, True),
                                            (1, 2, 64, 128, True), (3, 2, 1, 128, False), (1, 1, 130, 64, True),
                                            (2, 2, 128, 64, False), (1, 3, 384, 128, False), (2, 2, 515, 64, True), (1, 2, 577, 64, False),
                                            (2, 1, 256, 64, True), (1, 2, 1000, 64, True)])
def test_flash_attn(ops, B, H, S, D, causal, impl):
    """impl 1 = mma.sync kernel, 2 = wgmma kernel (two query warpgroups per CTA for Sq > 64), 3 = wgmma kernel with one
    query warpgroup per CTA only (all behind vsb_flash_attn_bf16)"""
    from vstar_b200 import _lib
    qkv = rnd(B * S, 3 * H * D, seed=40)
    _lib.call("vsb_attn_set_impl", impl)
    try:
        out = ops.attn_fused_qkv(qkv, B, S, H, D, causal, D ** -0.5)
        torch.cuda.synchronize()
    finally:
        _lib.call("vsb_attn_set_impl", 0)
    q, k, v = [t.transpose(1, 2).float() for t in qkv.view(B, S, 3, H, D).unbind(2)]
    att = q @ k.transpose(-1, -2) * D ** -0.5
    if causal:
        att = att + torch.full((S, S), float("-inf"), device="cuda").triu(1)
    ref = (torch.softmax(att, -1) @ v).transpose(1, 2).reshape(B * S, H * D)
    assert torch.allclose(out.float(), ref, rtol=2e-2, atol=2e-2), rel_err(out, ref)


@pytest.mark.parametrize("impl,Sq,Sk", [(1, 3, 100), (2, 3, 100), (2, 70, 300), (1, 70, 300), (4, 1, 100), (4, 3, 100), (4, 4, 383),
                                        (0, 1, 377), (4, 2, 9)])
def test_flash_attn_kv_cache_decode(ops, impl, Sq, Sk):
    """Sq < Sk with causal offset (decode / chunked prefill against a KV cache with a different row stride; cache rows
    beyond Sk hold NaNs and must never be read into the result); impl 4 = split-KV cluster decode kernel (auto for Sq <= 4)"""
    from vstar_b200 import _lib
    B, H, D, Tmax = 2, 4, 128, 384
    q = rnd(B * Sq, H * D, seed=41)
    kc, vc = rnd(B, Tmax, H * D, seed=42), rnd(B, Tmax, H * D, seed=43)
    kc[:, Sk:] = float("nan")
    vc[:, Sk:] = float("nan")
    out = torch.empty(B * Sq, H * D, dtype=BF, device="cuda")
    _lib.call("vsb_attn_set_impl", impl)
    try:
        ops.flash_attn(q, kc, vc, out, B, H, Sq, Sk, D, True, D ** -0.5, Sq * H * D, H * D, Tmax * H * D, H * D, Tmax * H * D, H * D,
                       Sq * H * D, H * D)
        torch.cuda.synchronize()
    finally:
        _lib.call("vsb_attn_set_impl", 0)
    qf = q.view(B, Sq, H, D).transpose(1, 2).float()
    kf = kc[:, :Sk].view(B, Sk, H, D).transpose(1, 2).float()
    vf = vc[:, :Sk].view(B, Sk, H, D).transpose(1, 2).float()
    att = qf @ kf.transpose(-1, -2) * D ** -0.5
    mask = torch.ones(Sq, Sk, device="cuda").tril(Sk - Sq).bool()
    att = att.masked_fill(~mask, float("-inf"))
    ref = (torch.softmax(att, -1) @ vf).transpose(1, 2).reshape(B * Sq, H * D)
    assert torch.allclose(out.float(), ref, rtol=2e-2, atol=2e-2), rel_err(out, ref)


@pytest.mark.parametrize("Nq,Nk,D", [(6, 2304, 16), (2304, 6, 16), (6, 6, 32)])
def test_attn_small(ops, Nq, Nk, D):
    B, H = 2, 8
    q, k, v = rnd(B * Nq, H * D, seed=50), rnd(B * Nk, H * D, seed=51), rnd(B * Nk, H * D, seed=52)
    out = ops.attn_small(q, k, v, B, H, Nq, Nk, D, 1 / math.sqrt(D))
    qf = q.view(B, Nq, H, D).transpose(1, 2).float()
    kf = k.view(B, Nk, H, D).transpose(1, 2).float()
    vf = v.view(B, Nk, H, D).transpose(1, 2).float()
    ref = (torch.softmax(qf @ kf.transpose(-1, -2) / math.sqrt(D), -1) @ vf).transpose(1, 2).reshape(B * Nq, H * D)
    assert torch.allclose(out.float(), ref, rtol=1e-2, atol=1e-2), rel_err(out, ref)


def test_embed_splice_gather_patchify_pos(ops):
    V, d, B, L, img_pos, n_img = 500, 256, 2, 20, 7, 16
    table = rnd(V, d, seed=60)
    ids = torch.randint(0, V, (B, L), device="cuda")
    ids[:, img_pos] = -200
    T = L - 1 + n_img
    out = torch.zeros(B, T, d, dtype=BF, device="cuda")
    ops.embed_splice(ids, table, out, img_pos, n_img)
    for b in range(B):
        assert torch.equal(out[b, :img_pos], table[ids[b, :img_pos]])
        assert torch.equal(out[b, img_pos + n_img:], table[ids[b, img_pos + 1:]])
        assert float(out[b, img_pos:img_pos + n_img].abs().max()) == 0
    idx = torch.tensor([3, 499, 0, 17], device="cuda")
    assert torch.equal(ops.gather_rows(idx, table), table[idx])
    # patchify == unfold with (c, py, px) ordering == conv weight.view(C_out, -1)
    Bi, S, P = 2, 56, 14
    px = rnd(Bi, 3, S, S, seed=61)
    A = ops.patchify(px, P, 592)
    ref = F.unfold(px.float(), kernel_size=P, stride=P).transpose(1, 2).reshape(-1, 3 * P * P)
    assert torch.equal(A[:, :588].float(), ref) and float(A[:, 588:].abs().max()) == 0
    x = rnd(Bi * 17, 64, seed=62)
    cls, pos = rnd(64, seed=63), rnd(17, 64, seed=64)
    y = ops.vit_add_pos_(x.clone(), cls, pos, Bi, 17).view(Bi, 17, 64)
    refy = torch.cat([cls.expand(Bi, 1, 64), x.view(Bi, 17, 64)[:, 1:]], 1) + pos
    assert torch.equal(y, refy)


def test_owl_merge_and_heads(ops):
    B, S, C, Q = 2, 2305, 128, 64
    x = rnd(B * S, C, seed=70)
    w1, b1, w2, b2 = [(1 + 0.1 * torch.randn(C)).to(BF).cuda() if i % 2 == 0 else rnd(C, scale=0.1, seed=71 + i) for i in range(4)]
    y = ops.owl_merge(x, w1, b1, w2, b2, B, S, 1e-5)
    xe = F.layer_norm(x.float().view(B, S, C), (C,), w1.float(), b1.float(), 1e-5).to(BF)
    m = (xe[:, 1:] * xe[:, :1])
    ref = F.layer_norm(m.float(), (C,), w2.float(), b2.float(), 1e-5)
    assert torch.allclose(y.view(B, S - 1, C).float(), ref, rtol=2e-2, atol=2e-2), rel_err(y.view(B, S - 1, C), ref)
    # class head epilogue
    R = B * 2304
    yy = torch.randn(R, Q + 2, device="cuda")
    query = rnd(B, Q, seed=75)
    logits, scores = ops.owl_class_post(yy, query, 2304, Q)
    e = yy[:, :Q].view(B, 2304, Q)
    e = e / (e.norm(dim=-1, keepdim=True) + 1e-6)
    qn = query.float() / (query.float().norm(dim=-1, keepdim=True) + 1e-6)
    lg = (torch.einsum("bpd,bd->bp", e, qn) + yy[:, Q].view(B, 2304)) * (F.elu(yy[:, Q + 1].view(B, 2304)) + 1)
    assert torch.allclose(logits.view(B, 2304), lg, rtol=1e-4, atol=1e-5)
    assert torch.allclose(scores.view(B, 2304), torch.sigmoid(lg), rtol=1e-4, atol=1e-5)
    bias = torch.randn(2304, 4, device="cuda")
    yb = torch.randn(R, 4, device="cuda")
    boxes = ops.owl_box_post(yb, bias, 2304)
    assert torch.allclose(boxes.view(B, 2304, 4), torch.sigmoid(yb.view(B, 2304, 4) + bias), rtol=1e-5, atol=1e-6)
    idx, val = ops.argmax_rows(logits.view(B, 2304))
    assert torch.equal(idx.long(), logits.view(B, 2304).argmax(-1))


def test_sam_upscale_helpers(ops):
    B, H, W, C = 2, 12, 12, 64
    x = rnd(B * H * W, C, seed=80)
    up = ops.upsample2x_nhwc(x, B, H, W, C)
    nchw = x.view(B, H, W, C).permute(0, 3, 1, 2).float()
    ref = F.interpolate(nchw, scale_factor=2.0, mode="bilinear").to(BF).permute(0, 2, 3, 1).reshape(-1, C)
    assert torch.equal(up, ref)
    A = ops.im2col3x3_nhwc(up, B, 2 * H, 2 * W, C)
    wconv = rnd(32, C, 3, 3, scale=0.05, seed=81)
    wperm = wconv.permute(0, 2, 3, 1).reshape(32, 9 * C).contiguous()
    out = ops.gemm(A, wperm, out_dtype=torch.float32)
    refc = F.conv2d(up.view(B, 2 * H, 2 * W, C).permute(0, 3, 1, 2).float(), wconv.float(), padding=1).permute(0, 2, 3, 1).reshape(-1, 32)
    assert torch.allclose(out, refc, rtol=1e-3, atol=1e-3), rel_err(out, refc)
    hyper = rnd(B, 32, seed=82)
    upb = out.to(BF).contiguous()
    md = ops.mask_dot(upb, hyper, B, 4 * H * W, 32)
    refm = torch.einsum("bpc,bc->bp", upb.view(B, -1, 32).float(), hyper.float())
    assert torch.allclose(md, refm, rtol=1e-4, atol=1e-4)
    a, bb = rnd(B * 10, 64, seed=83), rnd(10, 64, seed=84)
    assert torch.equal(ops.add_rows(a, bb).view(B, 10, 64), a.view(B, 10, 64) + bb)


@pytest.mark.parametrize("h,w", [(100, 120), (233, 96), (768, 768), (1023, 517), (2048, 2048)])
def test_heatmap_and_rect_sums(ops, h, w):
    low = torch.randn(192, 192, device="cuda") * 3
    hm, stats = ops.heatmap(low, h, w)
    ref = F.interpolate(low[None, None], (h, w), mode="bilinear", align_corners=False)[0, 0].clamp(min=0)
    assert torch.allclose(hm, ref, rtol=1e-5, atol=1e-5), rel_err(hm, ref)
    s = stats.cpu()
    assert abs(float(s[0]) - float(hm.max())) < 1e-6 and abs(float(s[1]) - float(hm.min())) < 1e-6
    assert abs(float(s[2]) - float(hm.double().sum())) <= 1e-5 * float(hm.double().sum()) + 1e-3
    rects = torch.tensor([[0, 0, w // 2, h // 2], [w // 2, 0, w - w // 2, h // 2], [0, h // 2, w // 2, h - h // 2],
                          [w // 2, h // 2, w - w // 2, h - h // 2], [0, 0, w, h], [3, 5, 1, 1]], dtype=torch.int32, device="cuda")
    sums = ops.rect_sums(hm, rects, stats).cpu()
    norm = ((hm - hm.min()) / (hm.max() - hm.min())).double()
    for i, (x0, y0, rw, rh) in enumerate(rects.cpu().tolist()):
        want = float(norm[y0:y0 + rh, x0:x0 + rw].sum())
        assert abs(float(sums[i]) - want) <= 1e-5 * abs(want) + 1e-4, (i, float(sums[i]), want)


@pytest.mark.parametrize("h,w,smallest", [(110, 150, 40), (512, 512, 100), (1900, 900, 300), (777, 1001, 251), (1024, 1024, 224)])
def test_crop_records_equal_materialised_path(ops, h, w, smallest):
    """vsb_pack_detections_f32 + vsb_heat_pyramids_f32 (no H x W map written) == heatmap + rect_sums + torch reductions,
    bit for bit: statistics, every rectangle sum of the quad-tree pyramid (cast to fp32 as the controller does), best
    score/box with first-index tie-break, count and compaction of the boxes above 0.5"""
    import numpy as np
    from vstar_b200 import records as RC
    g = torch.Generator(device="cuda").manual_seed(h * 7 + w)
    n, P = 3, 2304
    lows = torch.randn(n, 192, 192, device="cuda", generator=g) * 3
    scores = torch.rand(n, P, device="cuda", generator=g) * 0.45
    scores[0, 100], scores[0, 7], scores[0, 2000] = 0.9, 0.9, 0.6          # tie for the maximum: first index (7) must win
    scores[1, 40:70] = torch.linspace(0.95, 0.55, 30, device="cuda")        # 30 valid rows: only the first 16 are recorded
    boxes = torch.rand(n, P, 4, device="cuda", generator=g)
    bboxes = [[13, 29, w, h], [0, 0, w, h], [5, 0, w, h]]
    rects = [RC.pyramid_rects(b, smallest) for b in bboxes]
    rects[2] = []                                                          # a crop that is never split: no heat-map part
    R = RC.record_floats(max(len(r) for r in rects))
    rec = torch.zeros(n, R, device="cuda")
    ops.pack_detections(scores, boxes, rec)
    jobs = [(lows[i], h, w, [(r[0] - bboxes[i][0], r[1] - bboxes[i][1], r[2], r[3]) for r in rects[i]], i) for i in range(n) if rects[i]]
    ops.heat_pyramids(jobs, rec, 192, 192)
    rows = rec.cpu().numpy()
    for i in range(n):
        ti = int(scores[i].argmax())
        assert rows[i, RC.REC_TOPIDX] == ti and rows[i, RC.REC_TOP] == float(scores[i, ti]) and rows[i, RC.REC_NROWS] == P
        assert np.array_equal(rows[i, RC.REC_BOX:RC.REC_BOX + 4], boxes[i, ti].cpu().numpy())
        valid = (scores[i] > 0.5).nonzero().flatten()
        assert rows[i, RC.REC_NVALID] == len(valid)
        k = min(len(valid), RC.REC_MAXVALID)
        assert np.array_equal(rows[i, RC.REC_VALID:RC.REC_VALID + 4 * k].reshape(k, 4), boxes[i, valid[:k]].cpu().numpy())
        if not rects[i]:
            assert rows[i, RC.REC_NRECT] == 0
            continue
        hm, stats = ops.heatmap(lows[i].contiguous(), h, w)
        s = stats.cpu().numpy()
        assert rows[i, RC.REC_MAX] == s[0] == float(hm.max()) and rows[i, RC.REC_MIN] == s[1] == float(hm.min())
        assert abs(rows[i, RC.REC_SUM] - float(hm.double().sum())) <= 1e-5 * float(hm.double().sum()) + 1e-3
        assert rows[i, RC.REC_NRECT] == len(rects[i])
        rel = torch.tensor(jobs[[j[4] for j in jobs].index(i)][3], dtype=torch.int32, device="cuda")
        want = ops.rect_sums(hm, rel, stats).cpu().numpy().astype(np.float32)
        got = rows[i, RC.REC_PYR:RC.REC_PYR + len(rects[i])]
        assert np.array_equal(got, want), float(np.abs(got - want).max())
        # and against numpy: normalize_score per element in fp32 (IEEE division, like torch), float64 sums
        norm = ((hm - hm.min()) / (hm.max() - hm.min())).double().cpu().numpy()
        for (x, y, rw, rh), v in list(zip(jobs[[j[4] for j in jobs].index(i)][3], got))[:9]:
            assert abs(float(v) - norm[y:y + rh, x:x + rw].sum()) <= 2e-7 * norm[y:y + rh, x:x + rw].sum() + 1e-6
        ev = __import__("vstar_b200.visual_search", fromlist=["_NodeEval"])._NodeEval.from_record(rows[i], bboxes[i], smallest)
        assert ev.pyramid is not None and ev.pyramid.get(tuple(bboxes[i])) == float(got[0])
    # NaN scores: no finite maximum is reported instead of an out-of-range index (ADVICE r1)
    bad = torch.full((1, P), float("nan"), device="cuda")
    rec1 = torch.zeros(1, R, device="cuda")
    ops.pack_detections(bad, boxes[:1].contiguous(), rec1)
    assert float(rec1[0, RC.REC_TOPIDX]) == -1


def test_owl_head_epilogues_bf16_values(ops):
    """quant_bf16: logits / scores / boxes are bf16 VALUES (the reference model is bf16, visual_search.py:145): equal to
    rounding the fp32 results, and many rows tie at the maximum exactly as they do in the reference"""
    y = torch.randn(2 * 2304, 66, device="cuda")
    q = rnd(2, 64, seed=4)
    l0, s0 = ops.owl_class_post(y, q, 2304, 64)
    l1, s1 = ops.owl_class_post(y, q, 2304, 64, quant_bf16=True)
    assert torch.equal(l1, l0.to(BF).float()) and torch.equal(s1, s1.to(BF).float())
    assert float((s1 != torch.sigmoid(l1).to(BF).float()).float().mean()) < 1e-3       # expf vs torch's sigmoid: fp32 ulp at a bf16 tie
    yb = torch.randn(2304, 4, device="cuda")
    bias = torch.randn(2304, 4, device="cuda")
    b0 = ops.owl_box_post(yb, bias, 2304)
    b1 = ops.owl_box_post(yb, bias, 2304, quant_bf16=True)
    want = torch.sigmoid((yb.to(BF).float() + bias).to(BF).float()).to(BF).float()
    assert torch.equal(b1, b1.to(BF).float()) and float((b1 != want).float().mean()) < 1e-3 and float((b1 - b0).abs().max()) < 1.2e-2


def test_gemm_with_folded_rmsnorm(ops):
    """vsb_gemm_rowscale_bf16: (a) rstd applied in the epilogue == LlamaRMSNorm then GEMM up to bf16 rounding (the fused form skips
    two roundings of the activations), (b) the row statistics a producer leaves are the sums of squares of exactly the bf16 values
    it stored, (c) a chain producer -> consumer equals rmsnorm(x_new) @ W, (d) bit-identical rows for any M"""
    torch.manual_seed(1)
    M, d, inter = 700, 4096, 11008
    x = (torch.randn(M, d, device="cuda") * 1.5).to(BF)
    gamma = (1 + 0.1 * torch.randn(d, device="cuda")).to(BF)
    w = (torch.randn(1024, d, device="cuda") / math.sqrt(d)).to(BF)
    wf = (w.float() * gamma.float()[None, :]).to(BF)
    ref = ops.gemm(ops.rmsnorm(x, gamma, 1e-6), w)
    out = torch.empty(M, 1024, dtype=BF, device="cuda")
    ops.gemm_rowscale(x, wf, out, rowsq_in=ops.rowsq(x), eps=1e-6)
    assert rel_err(out, ref) < 1.5e-2
    want = ((x.float() * torch.rsqrt((x.float() ** 2).mean(-1, keepdim=True) + 1e-6)) @ wf.float().T)
    assert rel_err(out, want) < 6e-3                      # closer to exact arithmetic than the two-rounding reference form
    # producer: o-proj-like GEMM with residual, leaves row statistics of what it stored
    a = (torch.randn(M, d, device="cuda") * 0.5).to(BF)
    wo = (torch.randn(d, d, device="cuda") / math.sqrt(d)).to(BF)
    xn = x.clone()
    sq = torch.empty(d // 32, M, dtype=torch.float32, device="cuda")
    ops.gemm_rowscale(a, wo, xn, rowsq_out=sq, residual=xn)
    assert torch.equal(xn, ops.gemm(a, wo, residual=x.clone()))                       # same values as the plain GEMM
    want_sq = (xn.float() ** 2).view(M, d // 32, 32).sum(-1).T
    assert torch.allclose(sq, want_sq, rtol=1e-5, atol=1e-4)
    # consumer of those statistics (SwiGLU epilogue, interleaved gate/up rows)
    wgu = (torch.randn(2 * 512, d, device="cuda") / math.sqrt(d)).to(BF)
    wguf = (wgu.float() * gamma.float()[None, :]).to(BF)
    g1 = torch.empty(M, 512, dtype=BF, device="cuda")
    ops.gemm_rowscale(xn, wguf, g1, rowsq_in=sq, eps=1e-6, epilogue=ops.EPI_SWIGLU)
    g0 = ops.gemm(ops.rmsnorm(xn, gamma, 1e-6), wgu, epilogue=ops.EPI_SWIGLU)
    assert rel_err(g1, g0) < 2e-2
    for m in (5, 40, 300):                                                           # row results do not depend on M
        o2 = torch.empty(m, 512, dtype=BF, device="cuda")
        ops.gemm_rowscale(xn[:m].contiguous(), wguf, o2, rowsq_in=sq[:, :m].contiguous(), eps=1e-6, epilogue=ops.EPI_SWIGLU)
        assert torch.equal(o2, g1[:m])


def test_rows_invariant_to_batch(ops):
    """batch-invariant mode (vsb_set_batch_invariant): the first rows of a GEMM / RMSNorm are bit-identical whether the call
    carries 3, 16, 320, 2264 or 18112 rows - i.e. the wgmma tile variants (32/64/128/256 wide) accumulate every
    output element in the same order, and no row-count-dependent kernel family is taken.  This is what makes a crop's record
    independent of the batch it was evaluated in (speculative batching, frontier sharding)."""
    torch.manual_seed(0)
    x = (torch.randn(18112, 4096, device="cuda") * 0.5).to(BF)
    for N, K, epi in ((4096, 4096, ops.EPI_NONE), (22016, 4096, ops.EPI_SWIGLU), (512, 4096, ops.EPI_RELU), (32004, 4096, ops.EPI_NONE)):
        w = (torch.randn(N, K, device="cuda") / math.sqrt(K)).to(BF)
        fp32 = N == 32004
        with ops.batch_invariant():
            big = ops.gemm(x, w, epilogue=epi, out_dtype=torch.float32 if fp32 else BF)
            for m in (3, 16, 17, 320, 2264):
                y = ops.gemm(x[:m].contiguous(), w, epilogue=epi, out_dtype=torch.float32 if fp32 else BF)
                assert torch.equal(y, big[:m]), (N, epi, m, float((y.float() - big[:m].float()).abs().max()))
        # without the flag the skinny decode kernels take M <= 16: fast, but only equal up to bf16 rounding
        y3 = ops.gemm(x[:3].contiguous(), w, epilogue=epi, out_dtype=torch.float32 if fp32 else BF)
        assert rel_err(y3, big[:3]) < 2e-2
    g = (1 + 0.1 * torch.randn(4096, device="cuda")).to(BF)
    with ops.batch_invariant():
        big = ops.rmsnorm(x[:4096], g, 1e-6)
        for m in (1, 5, 32, 33):
            assert torch.equal(ops.rmsnorm(x[:m].contiguous(), g, 1e-6), big[:m])


def test_copy2d_and_cast(ops):
    src = rnd(50, 3 * 128, seed=90)
    dst = torch.zeros(50, 2 * 128, dtype=BF, device="cuda")
    ops.copy2d(src[:, 128:256], dst[:, 128:])
    assert torch.equal(dst[:, 128:], src[:, 128:256]) and float(dst[:, :128].abs().max()) == 0
    x = torch.randn(1000, device="cuda")
    assert torch.equal(ops.cast_f32_bf16(x), x.to(BF))


def test_ops_fail_loudly_on_cpu_tensors(ops):
    from vstar_b200._lib import VsbError
    with pytest.raises(VsbError):
        ops.gemm(torch.zeros(8, 8, dtype=BF), torch.zeros(8, 8, dtype=BF))


def test_llama_layers_native_runner(ops):
    """vsb_llama_layers (one native call for the whole stack) == the same kernels sequenced from Python, bit for bit,
    for a prefill (Tn = 70) followed by a decode step (Tn = 1, skinny GEMMs) on the fused-QKV cache"""
    d, H, inter, nl, B, Tmax = 256, 2, 512, 3, 2, 96
    hd = d // H
    layers = [dict(ln1=(1 + 0.1 * torch.randn(d)).to(BF).cuda(), wqkv=rnd(3 * d, d, scale=d ** -0.5, seed=70 + i),
                   wo=rnd(d, d, scale=d ** -0.5, seed=80 + i), ln2=(1 + 0.1 * torch.randn(d)).to(BF).cuda(),
                   wgu=rnd(2 * inter, d, scale=d ** -0.5, seed=90 + i), wdown=rnd(d, inter, scale=inter ** -0.5, seed=100 + i))
              for i in range(nl)]
    cos_t, sin_t = _rope_tables(Tmax, hd)
    table = ops.llama_layer_table(layers)

    def python_stack(x, cache, Tn, past):
        ld = 3 * d
        attn = torch.empty((B * Tn, d), dtype=BF, device="cuda")
        for li, L in enumerate(layers):
            h = ops.rmsnorm(x, L["ln1"], 1e-6)
            cl = cache[li].view(B * Tmax, ld)
            ops.gemm(h, L["wqkv"], out=cl, rows_per_group=Tn, group_stride=Tmax, group_offset=past)
            ops.rope_(cl, Tn, H, hd, cos_t, sin_t, pos0=past, rows=B * Tn, group_stride=Tmax, group_offset=past)
            ops.flash_attn(cl[past:], cl[:, d:], cl[:, 2 * d:], attn, B, H, Tn, past + Tn, hd, True, hd ** -0.5, Tmax * ld, ld, Tmax * ld, ld,
                           Tmax * ld, ld, Tn * d, d)
            ops.gemm(attn, L["wo"], out=x, residual=x)
            h = ops.rmsnorm(x, L["ln2"], 1e-6)
            gu = ops.gemm(h, L["wgu"], epilogue=ops.EPI_SWIGLU)
            ops.gemm(gu, L["wdown"], out=x, residual=x)
        return x

    def native_stack(x, cache, Tn, past):
        scratch = torch.empty(B * Tn * (2 * d + inter), dtype=BF, device="cuda")
        return ops.llama_layers(table, nl, x, B, Tn, past, cache, B, Tmax, d, H, inter, 1e-6, cos_t, sin_t, scratch)

    outs = []
    # (the native runner applies RoPE inside the QKV GEMM epilogue - head_dim 128 - while python_stack runs the separate kernel)
    for fn in (python_stack, native_stack):
        cache = torch.zeros(nl, B, Tmax, 3 * d, dtype=BF, device="cuda")
        x0 = rnd(B * 70, d, seed=110).clone()
        y0 = fn(x0, cache, 70, 0).clone()
        x1 = rnd(B * 1, d, seed=111).clone()
        y1 = fn(x1, cache, 1, 70).clone()
        outs.append((y0, y1, cache.clone()))
    torch.cuda.synchronize()
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)
    assert float(outs[0][0].float().abs().max()) > 0 and torch.isfinite(outs[0][1].float()).all()
    from vstar_b200 import _lib
    _lib.call("vsb_llama_set_fuse_rope", 0)                       # and with the fusion switched off: still the same bits
    try:
        cache = torch.zeros(nl, B, Tmax, 3 * d, dtype=BF, device="cuda")
        y0 = native_stack(rnd(B * 70, d, seed=110).clone(), cache, 70, 0)
        assert torch.equal(y0, outs[0][0])
    finally:
        _lib.call("vsb_llama_set_fuse_rope", 1)
    # tail mode: the last layer runs attention / o-proj / MLP over the last rows of every sequence only.  The cache (K/V of
    # every row, every layer) must be bit-identical; the tail rows are bit-identical when the compact GEMMs run on the same
    # wgmma tile kernels as the full pass (more than 16 rows: B * tail = 18) and equal to bf16 rounding when the few rows take
    # the decode GEMM kernels (B * tail = 10), whose k order differs.
    cache_f = torch.zeros(nl, B, Tmax, 3 * d, dtype=BF, device="cuda")
    xf = native_stack(rnd(B * 70, d, seed=110).clone(), cache_f, 70, 0)
    scratch = torch.empty(B * 70 * (2 * d + inter), dtype=BF, device="cuda")
    for tail, exact in ((9, True), (5, False)):
        cache_t = torch.zeros_like(cache_f)
        xt = rnd(B * 70, d, seed=110).clone()
        ops.llama_layers(table, nl, xt, B, 70, 0, cache_t, B, Tmax, d, H, inter, 1e-6, cos_t, sin_t, scratch, tail_rows=tail)
        torch.cuda.synchronize()
        assert torch.equal(cache_f, cache_t)
        a, b = xf.view(B, 70, d)[:, -tail:], xt.view(B, 70, d)[:, -tail:]
        if exact:
            assert torch.equal(a, b)
        assert torch.allclose(a.float(), b.float(), rtol=2e-2, atol=2e-2)
        assert not torch.equal(xf.view(B, 70, d)[:, :-tail], xt.view(B, 70, d)[:, :-tail])   # the other rows were indeed skipped
    with pytest.raises(Exception):
        native_stack(rnd(B * 30, d, seed=112), torch.zeros(nl, B, Tmax, 3 * d, dtype=BF, device="cuda"), 30, 70)    # exceeds Tmax
    # folded RMSNorm: ln1 / ln2 multiplied into wqkv / wgu, 1/rms applied in the GEMM epilogues (6 launches per layer).  Against the
    # unfused runner on the SAME folded weights (ln = 1): equal up to bf16 rounding; tail rows bit-identical to the full fused pass.
    ones = torch.ones(d, dtype=BF, device="cuda")
    folded = [dict(ln1=ones, ln2=ones, wqkv=(L["wqkv"].float() * L["ln1"].float()[None, :]).to(BF).contiguous(), wo=L["wo"],
                   wgu=(L["wgu"].float() * L["ln2"].float()[None, :]).to(BF).contiguous(), wdown=L["wdown"]) for L in layers]
    ftable = ops.llama_layer_table(folded)
    res = {}
    for fused in (False, True):
        cache = torch.zeros(nl, B, Tmax, 3 * d, dtype=BF, device="cuda")
        xx = rnd(B * 70, d, seed=110).clone()
        ops.llama_layers(ftable, nl, xx, B, 70, 0, cache, B, Tmax, d, H, inter, 1e-6, cos_t, sin_t, scratch, norm_folded=fused)
        res[fused] = (xx.clone(), cache.clone())
    torch.cuda.synchronize()
    assert rel_err(res[True][0], res[False][0]) < 3e-2 and rel_err(res[True][1], res[False][1]) < 3e-2
    assert rel_err(res[True][0], outs[1][0]) < 3e-2                                  # and to the un-folded weights with their norms
    cache_t = torch.zeros_like(cache_f)
    xt = rnd(B * 70, d, seed=110).clone()
    ops.llama_layers(ftable, nl, xt, B, 70, 0, cache_t, B, Tmax, d, H, inter, 1e-6, cos_t, sin_t, scratch, tail_rows=9, norm_folded=True)
    torch.cuda.synchronize()
    assert torch.equal(cache_t, res[True][1]) and torch.equal(xt.view(B, 70, d)[:, -9:], res[True][0].view(B, 70, d)[:, -9:])
