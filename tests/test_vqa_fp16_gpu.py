"""The SEAL VQA LLM in fp16, the reference's dtype (LLaVA/llava/model/builder.py:43), on the _f16 kernels.

(1) every _f16 entry point against an fp32 torch reference on the tiny config's shapes and on the real ones (Llama-7B d 4096,
    inter 11008, V 32000, T 600, decode B 1 / 8; CLIP 257 x 1024, 16 heads; perceiver 32 <-> 288 keys, 16 x 96), every GEMM and
    attention variant forced through the tuning hooks.  Criterion: err(kernel) <= 2 * err(torch's own fp16 computation) + ATOL,
    errors = max |x - ref| / max |ref|; plus the two bit-exactness properties of the bf16 kernels (fused QKV+RoPE == GEMM then
    RoPE, GEMM rows independent of M in batch-invariant mode) and the native layer runner == the same kernels from Python.
(2) the fp16 engine against the reference goldens (tests/golden/vqa_a_*.npz, fp32): logits within 2 x the fp16 oracle's error
    + 1e-3, option NLLs within 2e-3 (the bf16 engine is allowed 5e-2), the same option / greedy ids wherever the reference's
    margins exceed the error.  fp16 and bf16 engine errors are written side by side to the JSON report.
(3) the rest of the VQA surface in fp16: continuous-batched decode, batched option scoring, device pixels, the model adapter
    with .half() inputs, a streamed safetensors checkpoint, and seal_answer next to the bf16 VSM."""
import json
import math
import os

import numpy as np
import pytest
import torch

from tests.helpers import REPORT_DIR

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
BF, F16 = torch.bfloat16, torch.float16
ATOL = 2e-3          # relative to max |ref|: fp16 output rounding is 2^-11 = 4.9e-4 of a value


@pytest.fixture(scope="module")
def ops():
    from vstar_b200 import ops as o
    return o


def rnd(*shape, scale=1.0, seed=0, dtype=F16):
    g = torch.Generator(device="cpu").manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def err(a, ref):
    a, ref = a.float(), ref.float().to(a.device)
    return float((a - ref).abs().max() / (ref.abs().max() + 1e-12))


def check(got, ref32, torch16, what):
    e, et = err(got, ref32), err(torch16, ref32)
    assert e <= 2 * et + ATOL, (what, e, et)
    return e, et


def tuned(force_bn):
    from vstar_b200 import _lib

    class Ctx:
        def __enter__(self):
            _lib.call("vsb_gemm_set_tuning", force_bn, 0)

        def __exit__(self, *a):
            _lib.call("vsb_gemm_set_tuning", 0, 0)
    return Ctx()


def attn_impl(impl):
    from vstar_b200 import _lib

    class Ctx:
        def __enter__(self):
            _lib.call("vsb_attn_set_impl", impl)

        def __exit__(self, *a):
            _lib.call("vsb_attn_set_impl", 0)
    return Ctx()


# ------------------------------------------------------------------------------------------------ (1) kernels
# (M, N, K, epilogue): Llama-7B prefill T = 600 / decode B = 1, 8 / lm_head; CLIP-L 257 rows; tiny config (d 256, inter 512)
GEMMS = [(600, 12288, 4096, "none"), (600, 4096, 11008, "res"), (600, 22016, 4096, "swiglu"), (8, 32000, 4096, "fp32"),
         (1, 12288, 4096, "none"), (8, 22016, 4096, "swiglu"), (1, 4096, 11008, "res"), (257, 3072, 1024, "bias"),
         (257, 4096, 1024, "quick_gelu"), (257, 1024, 4096, "bias_res"), (32, 1024, 1024, "gelu"), (70, 768, 256, "none"),
         (5, 1024, 256, "swiglu"), (3, 320, 256, "fp32")]


def _gemm_case(ops, M, N, K, epi, force):
    a, w = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2)
    b, r = rnd(N, scale=0.1, seed=3), rnd(M, N, seed=4)
    kw, code = {}, ops.EPI_NONE
    if "bias" in epi:
        kw["bias"] = b
    if "res" in epi:
        kw["residual"] = r
    if epi == "fp32":
        kw["out_dtype"] = torch.float32
    code = dict(quick_gelu=ops.EPI_QUICK_GELU, gelu=ops.EPI_GELU, swiglu=ops.EPI_SWIGLU).get(epi, ops.EPI_NONE)
    with tuned(force):
        out = ops.gemm(a, w, epilogue=code, **kw)
    torch.cuda.synchronize()

    def ref(dt):
        y = (a.to(dt) @ w.to(dt).t())
        if "bias" in kw:
            y = y + b.to(dt)
        if code == ops.EPI_QUICK_GELU:
            y = y * torch.sigmoid(1.702 * y)
        elif code == ops.EPI_GELU:
            y = torch.nn.functional.gelu(y)
        elif code == ops.EPI_SWIGLU:
            y = torch.nn.functional.silu(y[:, 0::2]) * y[:, 1::2]
        if "residual" in kw:
            y = y + r.to(dt)
        return y
    return check(out, ref(torch.float32), ref(F16), (M, N, K, epi, force))


@pytest.mark.parametrize("M,N,K,epi", GEMMS)
def test_gemm_f16_auto(ops, M, N, K, epi):
    _gemm_case(ops, M, N, K, epi, 0)


@pytest.mark.parametrize("force", [1, 2, 32, 64, 128, 256])
def test_gemm_f16_forced_variants(ops, force):
    """every kernel behind vsb_gemm_f16: the two skinny decode kernels (1: M <= 8, 2: M <= 16) and the 4 wgmma tile widths"""
    shapes = [(8, 4096, 4096, "res"), (1, 22016, 4096, "swiglu"), (5, 1024, 256, "bias")] if force == 1 else \
        [(16, 4096, 4096, "res"), (8, 22016, 4096, "swiglu"), (5, 1024, 256, "bias")] if force == 2 else \
        [(600, 4096, 4096, "res"), (600, 22016, 4096, "swiglu"), (257, 4096, 1024, "quick_gelu"), (70, 768, 256, "fp32")]
    for M, N, K, epi in shapes:
        _gemm_case(ops, M, N, K, epi, force)


def test_gemm_f16_rejects_mixed_dtypes(ops):
    from vstar_b200._lib import VsbError
    a, w = rnd(16, 64, seed=5), rnd(32, 64, seed=6)
    with pytest.raises(VsbError):
        ops.gemm(a.to(BF), w)
    with pytest.raises(VsbError):
        ops.gemm(a, w, bias=rnd(32, seed=7, dtype=BF))
    with pytest.raises(VsbError):
        ops.rmsnorm(a, torch.ones(64, dtype=BF, device="cuda"), 1e-6)
    with pytest.raises(VsbError):
        ops.attn_small(a, a, a.to(BF), 1, 1, 16, 16, 64, 0.1)


def _rope_tables(maxpos, D, dtype=F16, theta=10000.0):
    inv = 1.0 / (theta ** (torch.arange(0, D, 2, dtype=torch.float32) / D))
    fr = torch.outer(torch.arange(maxpos, dtype=torch.float32), inv)
    return fr.cos().to(dtype).cuda(), fr.sin().to(dtype).cuda()


def _rot(x):
    D = x.shape[-1]
    return torch.cat([-x[..., D // 2:], x[..., :D // 2]], -1)


@pytest.mark.parametrize("T,H", [(37, 2), (600, 32)])
def test_rope_f16_bit_exact_hf(ops, T, H):
    """RoPE in fp16 == HF's fp16 ops on fp16 tables: q * cos + rotate_half(q) * sin, every product and the sum rounded to fp16"""
    B, D = 2, 128
    qkv = rnd(B * T, 3 * H * D, seed=30)
    cos_t, sin_t = _rope_tables(max(64, T), D)
    cos = torch.cat([cos_t[:T], cos_t[:T]], -1)[None, :, None, :]
    sin = torch.cat([sin_t[:T], sin_t[:T]], -1)[None, :, None, :]
    ref = qkv.clone().view(B, T, 3, H, D)
    for i in (0, 1):
        x = ref[:, :, i]
        ref[:, :, i] = (x * cos) + (_rot(x) * sin)
    out = ops.rope_(qkv.clone(), T, H, D, cos_t, sin_t)
    assert torch.equal(out.view(B, T, 3, H, D), ref)


def test_gemm_qkv_rope_f16_equals_gemm_then_rope(ops):
    """vsb_gemm_qkv_rope_f16 (RoPE in the GEMM epilogue) is bit-identical to vsb_gemm_f16 followed by vsb_rope_f16, with and
    without the folded RMSNorm row scale (== vsb_gemm_rowscale_f16 followed by vsb_rope_f16)"""
    from vstar_b200 import _lib
    for d, T, B in ((256, 70, 2), (4096, 600, 1)):
        H, hd = d // 128, 128
        x, w = rnd(B * T, d, seed=11), rnd(3 * d, d, scale=d ** -0.5, seed=12)
        cos_t, sin_t = _rope_tables(1024, hd)
        sq = ops.rowsq(x)
        for folded in (False, True):
            ref = torch.empty(B * T, 3 * d, dtype=F16, device="cuda")
            if folded:
                ops.gemm_rowscale(x, w, ref, rowsq_in=sq, eps=1e-6)
            else:
                ops.gemm(x, w, out=ref)
            ops.rope_(ref, T, H, hd, cos_t, sin_t, pos0=5)
            out = torch.empty_like(ref)
            _lib.call("vsb_gemm_qkv_rope_f16", x.data_ptr(), d, w.data_ptr(), d, out.data_ptr(), 3 * d, B * T, 3 * d, d, 0, 0, 0,
                      sq.data_ptr() if folded else 0, 1, 1e-6, B * T, cos_t.data_ptr(), sin_t.data_ptr(), 0, T, 5, hd, ops._stream())
            torch.cuda.synchronize()
            assert torch.equal(out, ref), (d, folded)


def test_rows_invariant_to_batch_f16(ops):
    """batch-invariant mode: the first rows of an f16 GEMM / RMSNorm are bit-identical whatever the row count of the call"""
    torch.manual_seed(0)
    x = (torch.randn(2264, 4096, device="cuda") * 0.5).to(F16)
    for N, K, epi in ((4096, 4096, ops.EPI_NONE), (22016, 4096, ops.EPI_SWIGLU), (32000, 4096, None)):
        w = (torch.randn(N, K, device="cuda") / math.sqrt(K)).to(F16)
        kw = dict(out_dtype=torch.float32) if epi is None else dict(epilogue=epi)
        with ops.batch_invariant():
            big = ops.gemm(x, w, **kw)
            for m in (3, 16, 17, 320):
                y = ops.gemm(x[:m].contiguous(), w, **kw)
                assert torch.equal(y, big[:m]), (N, m)
    g = (1 + 0.1 * torch.randn(4096, device="cuda")).to(F16)
    with ops.batch_invariant():
        big = ops.rmsnorm(x, g, 1e-6)
        for m in (1, 5, 32, 33):
            assert torch.equal(ops.rmsnorm(x[:m].contiguous(), g, 1e-6), big[:m])


@pytest.mark.parametrize("rows,cols", [(600, 4096), (8, 4096), (1, 4096), (257, 1024), (70, 256), (288, 1024)])
def test_norms_rowsq_add_cast_f16(ops, rows, cols):
    F = torch.nn.functional
    x = rnd(rows, cols, seed=20)
    w, b = (1 + 0.1 * rnd(cols, seed=21, dtype=torch.float32)).to(F16), rnd(cols, scale=0.1, seed=22)
    # LayerNorm (fp32 statistics) with and without the fused GELU
    for act in (ops.EPI_NONE, ops.EPI_GELU):
        y = ops.layernorm(x, w, b, 1e-5, act=act)

        def ln(dt):
            o = F.layer_norm(x.to(dt), (cols,), w.to(dt), b.to(dt), 1e-5)
            return F.gelu(o) if act == ops.EPI_GELU else o
        check(y, ln(torch.float32), ln(F16), ("layernorm", act))
    # LlamaRMSNorm as HF computes it in fp16: fp32 statistics, rounded to fp16, times the fp16 weight
    y = ops.rmsnorm(x, w, 1e-6)
    xf = x.float()
    hs = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6)
    check(y, w.float() * hs, w * hs.to(F16), "rmsnorm")
    assert torch.allclose(ops.rowsq(x)[0], xf.pow(2).sum(-1), rtol=1e-4, atol=1e-3)
    p = rnd(3, cols, seed=23)
    ya = ops.add_rows(x, p)
    idx = torch.arange(rows, device="cuda") % 3
    assert torch.equal(ya, x + p[idx])                      # one fp16 rounding of the fp32 sum == torch's fp16 add
    f = torch.randn(rows, cols, device="cuda") * 3
    assert torch.equal(ops.cast_f32(f, F16), f.half())


def test_vit_add_pos_and_copies_f16(ops):
    B, S, C = 2, 257, 1024
    x = rnd(B * S, C, seed=24)
    cls, pos = rnd(C, seed=25), rnd(S, C, seed=26)
    ref = x.clone().view(B, S, C)
    ref[:, 0] = cls
    ref = ref + pos[None]
    y = ops.vit_add_pos_(x.clone(), cls, pos, B, S)
    assert torch.equal(y.view(B, S, C), ref)
    # pure 2-byte copies serve fp16 as they are
    px = rnd(2, 3, 224, 224, seed=27)
    A = ops.patchify(px, 14, 592)
    assert A.dtype == F16 and torch.equal(A[:, :588], px.view(2, 3, 16, 14, 16, 14).permute(0, 2, 4, 1, 3, 5).reshape(512, 588))
    idx = torch.tensor([3, 0, 7], dtype=torch.int64, device="cuda")
    assert torch.equal(ops.gather_rows(idx, x), x[idx])


def _attn_ref(q, k, v, scale, mask=None):
    """(fp32 reference, torch's fp16 computation as HF: scores in fp16, softmax in fp32 -> fp16, P @ V in fp16)"""
    out = []
    for dt in (torch.float32, F16):
        s = (q.to(dt) @ k.to(dt).transpose(-1, -2)) * scale
        if mask is not None:
            s = s.masked_fill(~mask, float("-inf"))
        p = torch.softmax(s, -1, dtype=torch.float32).to(dt)
        out.append(p @ v.to(dt))
    return out


@pytest.mark.parametrize("impl", [0, 1, 2, 3])
@pytest.mark.parametrize("B,H,S,D,causal", [(2, 16, 257, 64, False), (1, 32, 600, 128, True), (2, 2, 70, 128, True), (1, 2, 257, 64, False)])
def test_flash_attn_f16(ops, B, H, S, D, causal, impl):
    """CLIP-L (257 tokens, 16 x 64), Llama-7B prefill (600, 32 x 128, causal) and the tiny config; impl 1 = mma.sync,
    2 = wgmma (two query warpgroups per CTA), 3 = wgmma with one query warpgroup per CTA, 0 = auto"""
    qkv = rnd(B * S, 3 * H * D, seed=40)
    with attn_impl(impl):
        out = ops.attn_fused_qkv(qkv, B, S, H, D, causal, D ** -0.5)
        torch.cuda.synchronize()
    q, k, v = [t.transpose(1, 2) for t in qkv.view(B, S, 3, H, D).unbind(2)]
    mask = torch.ones(S, S, device="cuda").tril().bool() if causal else None
    r32, r16 = [r.transpose(1, 2).reshape(B * S, H * D) for r in _attn_ref(q, k, v, D ** -0.5, mask)]
    check(out, r32, r16, (B, H, S, D, causal, impl))


@pytest.mark.parametrize("impl,B,Sq,Sk", [(4, 1, 1, 600), (4, 8, 1, 600), (0, 8, 1, 600), (4, 2, 3, 100), (1, 2, 3, 100), (2, 1, 70, 600)])
def test_attn_decode_f16(ops, impl, B, Sq, Sk):
    """decode against the KV cache (Llama-7B, 32 x 128, B 1 and 8): split-KV cluster kernel (impl 4 / auto) and the others on a
    strided cache whose rows beyond Sk hold NaNs; plus vsb_attn_decode_f16 with left-padded ragged sequences (k_start)"""
    from vstar_b200 import _lib
    H, D, Tmax = 32, 128, 640
    q = rnd(B * Sq, H * D, seed=41)
    kc, vc = rnd(B, Tmax, H * D, seed=42), rnd(B, Tmax, H * D, seed=43)
    kc[:, Sk:] = float("nan")
    vc[:, Sk:] = float("nan")
    out = torch.empty(B * Sq, H * D, dtype=F16, device="cuda")
    with attn_impl(impl):
        ops.flash_attn(q, kc, vc, out, B, H, Sq, Sk, D, True, D ** -0.5, Sq * H * D, H * D, Tmax * H * D, H * D, Tmax * H * D, H * D,
                       Sq * H * D, H * D)
        torch.cuda.synchronize()
    qf = q.view(B, Sq, H, D).transpose(1, 2)
    kf, vf = [t[:, :Sk].reshape(B, Sk, H, D).transpose(1, 2) for t in (kc, vc)]
    mask = torch.ones(Sq, Sk, device="cuda").tril(Sk - Sq).bool()
    r32, r16 = [r.transpose(1, 2).reshape(B * Sq, H * D) for r in _attn_ref(qf, kf, vf, D ** -0.5, mask)]
    check(out, r32, r16, (impl, B, Sq, Sk))
    if Sq == 1 and B > 1:
        k_start = torch.tensor([(37 * b) % 200 for b in range(B)], dtype=torch.int32, device="cuda")
        o2 = torch.empty_like(out)
        _lib.call("vsb_attn_decode_f16", q.data_ptr(), kc.data_ptr(), vc.data_ptr(), o2.data_ptr(), H * D, H * D, Tmax * H * D, H * D,
                  Tmax * H * D, H * D, H * D, H * D, B, H, 1, Sk, D, 1, D ** -0.5, k_start.data_ptr(), ops._stream())
        torch.cuda.synchronize()
        for b in range(B):
            s0 = int(k_start[b])
            r32, r16 = _attn_ref(qf[b:b + 1], kf[b:b + 1, :, s0:], vf[b:b + 1, :, s0:], D ** -0.5)
            check(o2[b], r32.reshape(-1), r16.reshape(-1), ("ragged", b))


@pytest.mark.parametrize("H", [2, 32])
def test_flash_attn_seg_f16(ops, H):
    """answer-option scoring: 4 options appended back to back after a 600-row prefix, each row sees the prefix and its own option"""
    from vstar_b200 import _lib
    D, P, lens = 128, 600, [3, 5, 2, 6]
    Sq = sum(lens)
    Sk = P + Sq
    q = rnd(Sq, H * D, seed=44)
    kc, vc = rnd(Sk, H * D, seed=45), rnd(Sk, H * D, seed=46)
    seg, mask = [], torch.zeros(Sq, Sk, dtype=torch.bool)
    r0 = 0
    for n in lens:
        for j in range(n):
            seg.append(P + r0)
            mask[r0 + j, :P] = True
            mask[r0 + j, P + r0:P + r0 + j + 1] = True
        r0 += n
    seg = torch.tensor(seg, dtype=torch.int32, device="cuda")
    out = torch.empty(Sq, H * D, dtype=F16, device="cuda")
    _lib.call("vsb_flash_attn_seg_f16", q.data_ptr(), kc.data_ptr(), vc.data_ptr(), out.data_ptr(), Sq * H * D, H * D, Sk * H * D, H * D,
              Sk * H * D, H * D, Sq * H * D, H * D, 1, H, Sq, Sk, D, D ** -0.5, seg.data_ptr(), P, ops._stream())
    torch.cuda.synchronize()
    qf, kf, vf = [t.view(-1, H, D).transpose(0, 1) for t in (q, kc, vc)]
    r32, r16 = [r.transpose(0, 1).reshape(Sq, H * D) for r in _attn_ref(qf, kf, vf, D ** -0.5, mask.cuda())]
    check(out, r32, r16, ("seg", H))


def test_attn_small_f16_perceiver(ops):
    """perceiver resampler attention: 16 heads x 96, 32 latents against 288 keys (256 patches + 32 latents), 3 crops"""
    B, H, D, Nq, Nk = 3, 16, 96, 32, 288
    q, kv = rnd(B * Nq, H * D, seed=50), rnd(B * Nk, 2 * H * D, seed=51)
    out = ops.attn_small(q, kv[:, :H * D], kv[:, H * D:], B, H, Nq, Nk, D, D ** -0.5)
    qf = q.view(B, Nq, H, D).transpose(1, 2)
    kf = kv[:, :H * D].reshape(B, Nk, H, D).transpose(1, 2)
    vf = kv[:, H * D:].reshape(B, Nk, H, D).transpose(1, 2)
    r32, r16 = [r.transpose(1, 2).reshape(B * Nq, H * D) for r in _attn_ref(qf, kf, vf, D ** -0.5)]
    check(out, r32, r16, "attn_small")


def test_llama_layers_f16_native_runner(ops):
    """vsb_llama_layers_f16 == the same f16 kernels sequenced from Python, bit for bit (prefill Tn = 70, then a decode step), and
    the folded-RMSNorm runner on folded weights within fp16 rounding of it"""
    d, H, inter, nl, B, Tmax = 256, 2, 512, 3, 2, 96
    hd = d // H
    layers = [dict(ln1=(1 + 0.1 * torch.randn(d)).to(F16).cuda(), wqkv=rnd(3 * d, d, scale=d ** -0.5, seed=70 + i),
                   wo=rnd(d, d, scale=d ** -0.5, seed=80 + i), ln2=(1 + 0.1 * torch.randn(d)).to(F16).cuda(),
                   wgu=rnd(2 * inter, d, scale=d ** -0.5, seed=90 + i), wdown=rnd(d, inter, scale=inter ** -0.5, seed=100 + i))
              for i in range(nl)]
    cos_t, sin_t = _rope_tables(Tmax, hd)
    table = ops.llama_layer_table(layers)

    def python_stack(x, cache, Tn, past):
        ld = 3 * d
        attn = torch.empty((B * Tn, d), dtype=F16, device="cuda")
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

    def native_stack(x, cache, Tn, past, tab=table, folded=False):
        scratch = torch.empty(B * Tn * (2 * d + inter), dtype=F16, device="cuda")
        return ops.llama_layers(tab, nl, x, B, Tn, past, cache, B, Tmax, d, H, inter, 1e-6, cos_t, sin_t, scratch, norm_folded=folded)

    outs = []
    for fn in (python_stack, native_stack):
        cache = torch.zeros(nl, B, Tmax, 3 * d, dtype=F16, device="cuda")
        y0 = fn(rnd(B * 70, d, seed=110).clone(), cache, 70, 0).clone()
        y1 = fn(rnd(B * 1, d, seed=111).clone(), cache, 1, 70).clone()
        outs.append((y0, y1, cache.clone()))
    torch.cuda.synchronize()
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)
    assert torch.isfinite(outs[0][0].float()).all() and float(outs[0][0].float().abs().max()) > 0
    ones = torch.ones(d, dtype=F16, device="cuda")
    folded = [dict(ln1=ones, ln2=ones, wqkv=(L["wqkv"].float() * L["ln1"].float()[None, :]).to(F16).contiguous(), wo=L["wo"],
                   wgu=(L["wgu"].float() * L["ln2"].float()[None, :]).to(F16).contiguous(), wdown=L["wdown"]) for L in layers]
    cache = torch.zeros(nl, B, Tmax, 3 * d, dtype=F16, device="cuda")
    yf = native_stack(rnd(B * 70, d, seed=110).clone(), cache, 70, 0, tab=ops.llama_layer_table(folded), folded=True)
    torch.cuda.synchronize()
    assert err(yf, outs[0][0]) < 5e-3
    with pytest.raises(Exception):                       # weights of one dtype, activations of the other
        native_stack(rnd(B * 70, d, seed=110, dtype=BF), torch.zeros(nl, B, Tmax, 3 * d, dtype=BF, device="cuda"), 70, 0)


# ------------------------------------------------------------------------------------------------ (2) engine parity
@pytest.fixture(scope="module")
def setup():
    from oracle import vqa_oracle as V, vsm_oracle as O
    from vstar_b200 import synth
    from vstar_b200.vqa import VQAEngine, VQAWeights
    cfg = O.tiny_config()
    sd = {k: synth.synthetic_tensor(k, shp, seed=4321) for k, shp in V.vqa_state_dict_shapes(cfg).items()}
    eng = VQAEngine(VQAWeights.from_state_dict(cfg, sd, dtype=F16), max_tokens=1024)
    assert eng.dtype == F16 and eng.w.lm_head.dtype == F16 and eng.w.rope_cos.dtype == F16
    return V, O, cfg, sd, eng


@pytest.fixture(scope="module")
def bf16_engine(setup):
    from vstar_b200.vqa import VQAEngine, VQAWeights
    V, O, cfg, sd, _ = setup
    return VQAEngine(VQAWeights.from_state_dict(cfg, sd), max_tokens=1024)


def inputs(g):
    gen = torch.Generator().manual_seed(int(g["img_seed"]))
    image = torch.randn(1, 3, 224, 224, generator=gen)
    crops = torch.randn(2, 3, 224, 224, generator=gen)
    q = torch.from_numpy(g["q"])
    opts, o = [], 0
    for n in g["opt_lens"]:
        opts.append(torch.from_numpy(g["opts"][o:o + int(n)]))
        o += int(n)
    return image, crops, q, opts, [bool(x) for x in g["images_long"]], [bool(x) for x in g["objects_long"]]


def _engine_errors(eng, dt, q, image, crops, il, ol, opts, l32, ref_l):
    ic, cc = image.to(dt).cuda(), crops.to(dt).cuda()
    x = eng.build_embeds(q[0].tolist(), ic, cc, il, ol)
    T = x.shape[0]
    eng.prefill_embeds(x)
    _, am, logits = eng._logits_rows(x, torch.arange(T, device="cuda"))
    losses, choice = eng.option_losses(q[0].tolist(), [o.tolist() for o in opts], ic, cc, il, ol)
    return err(logits, l32[0]), float((losses - ref_l).abs().max()), am.cpu().long(), losses, choice, (ic, cc)


@pytest.mark.parametrize("sub", ["short_long", "long_short"])
def test_fp16_engine_parity_on_goldens(setup, bf16_engine, sub):
    V, O, cfg, sd, eng = setup
    g = np.load(os.path.join(G, f"vqa_a_{sub}.npz"))
    image, crops, q, opts, il, ol = inputs(g)
    e32 = V.build_embeds(sd, cfg, q, image, crops, il, ol)
    l32 = V.forward_logits(sd, cfg, e32)
    assert err(l32[0, -1], torch.from_numpy(g["logits_last"])) < 1e-4
    sd16 = {k: v.half() for k, v in sd.items()}
    l16 = V.forward_logits(sd16, cfg, V.build_embeds(sd16, cfg, q, image.half(), crops.half(), il, ol))
    e_oracle16 = err(l16[0], l32[0])
    ref_l = torch.from_numpy(g["option_losses"])
    e16, nll16, am, losses, choice, (ic, cc) = _engine_errors(eng, F16, q, image, crops, il, ol, opts, l32, ref_l)
    e_bf, nll_bf, _, losses_bf, choice_bf, _ = _engine_errors(bf16_engine, BF, q, image, crops, il, ol, opts, l32, ref_l)
    assert e16 <= 2 * e_oracle16 + 1e-3, (e16, e_oracle16)
    assert nll16 < 2e-3, (losses, ref_l)
    srt = ref_l.sort().values
    if float(srt[1] - srt[0]) > 2 * 2e-3:
        assert choice == int(ref_l.argmin())
    top2 = l32[0].topk(2, dim=-1).values
    confident = (top2[:, 0] - top2[:, 1]) > 1e-2
    assert torch.equal(am[confident], torch.from_numpy(g["logits_argmax"])[confident])
    # greedy generation: the golden ids wherever the fp32 reference's top-2 gap along the golden path exceeds 1e-2
    gold = g["gen"].tolist()
    out = eng.generate(q[0].tolist(), ic, cc, il, ol, max_new_tokens=len(gold), eos_token_id=-1)
    emb = sd["model.embed_tokens.weight"]
    embeds = e32.clone()
    for t, (mine, ref_t) in enumerate(zip(out, gold)):
        last = V.forward_logits(sd, cfg, embeds)[0, -1]
        gap = float(last.topk(2).values[0] - last.topk(2).values[1])
        if gap > 1e-2:
            assert mine == ref_t, (t, out, gold, gap)
        if mine != ref_t:
            break                                   # a near-tie went the other way: the paths differ from here on
        embeds = torch.cat([embeds, emb[torch.tensor([ref_t])].unsqueeze(0)], dim=1)
    json.dump(dict(fp16=dict(logits_err=e16, nll_err=nll16, losses=losses.tolist(), choice=choice, gen=out),
                   bf16=dict(logits_err=e_bf, nll_err=nll_bf, losses=losses_bf.tolist(), choice=choice_bf),
                   fp16_oracle_logits_err=e_oracle16, ref_losses=ref_l.tolist(), ref_gen=gold),
              open(os.path.join(REPORT_DIR, f"vqa_fp16_parity_{sub}.json"), "w"), indent=1)
    assert e16 < e_bf and nll16 < nll_bf, (e16, e_bf, nll16, nll_bf)


# ------------------------------------------------------------------------------------------------ (3) the rest of the surface
def rel(a, b):
    return err(torch.as_tensor(a).cpu(), torch.as_tensor(b).cpu())


def test_continuous_batched_decode_f16(setup):
    """prefill_ragged / decode_ragged / generate_batch in fp16 against the single-sequence path and the fp32 oracle (the per-step
    check of the bf16 test)"""
    V, O, cfg, sd, eng = setup
    rng = np.random.default_rng(5)
    gen = torch.Generator().manual_seed(7)
    reqs, embeds32 = [], []
    for n_pre, n_post, long_ in ((5, 9, True), (12, 30, False), (3, 4, True)):
        ids = [1] + rng.integers(3, cfg.vocab - 30, n_pre).tolist() + [-200] + rng.integers(3, cfg.vocab - 30, n_post).tolist()
        image = torch.randn(1, 3, 224, 224, generator=gen)
        reqs.append((ids, image.to(F16).cuda(), None, [long_], None))
        embeds32.append(V.build_embeds(sd, cfg, torch.tensor([ids]), image, None, [long_], None))
    forced = [[7, 11, 13], [17, 19, 23], [29, 31, 37]]
    single = []
    for (ids, img, _, il, _), f in zip(reqs, forced):
        x = eng.build_embeds(ids, img, None, il, None)
        T = x.shape[0]
        eng.prefill_embeds(x)
        rows = [eng.last_logits(x)[0].clone()]
        for s_, t in enumerate(f):
            rows.append(eng.append_tokens([t], T + s_)[0].clone())
        single.append(torch.stack(rows))
    xs = [eng.build_embeds(ids, img, None, il, None) for ids, img, _, il, _ in reqs]
    logits, Tpad, lens = eng.prefill_ragged(xs)
    assert lens == [e.shape[1] for e in embeds32] and Tpad == max(lens)
    batch_rows = [logits.clone()]
    for s_ in range(3):
        batch_rows.append(eng.decode_ragged([f[s_] for f in forced], lens, Tpad, s_).clone())
    emb = sd["model.embed_tokens.weight"]
    for b in range(3):
        got = torch.stack([r[b] for r in batch_rows])
        e = embeds32[b].clone()
        for s_ in range(4):
            ref = V.forward_logits(sd, cfg, e)[0, -1]
            assert rel(got[s_], ref) < 3e-2 and rel(single[b][s_], ref) < 3e-2, (b, s_, rel(got[s_], ref))
            assert rel(got[s_], single[b][s_]) < 3e-2
            if s_ < 3:
                e = torch.cat([e, emb[torch.tensor([forced[b][s_]])].unsqueeze(0)], dim=1)
    outs = eng.generate_batch(reqs, max_new_tokens=4, eos_token_id=-1)
    assert [len(o) for o in outs] == [4, 4, 4]
    for b in range(3):
        e = embeds32[b].clone()
        for t in outs[b]:
            last = V.forward_logits(sd, cfg, e)[0, -1]
            assert float(last.max() - last[t]) < 3e-2
            e = torch.cat([e, emb[torch.tensor([t])].unsqueeze(0)], dim=1)


def test_option_losses_batch_f16(setup):
    """several questions in one option-scoring pass == one question at a time (fp16 rounding level for the batched group)"""
    V, O, cfg, sd, eng = setup
    items = []
    for sub in ("short_long", "long_short", "short_long"):
        g = np.load(os.path.join(G, f"vqa_a_{sub}.npz"))
        image, crops, q, opts, il, ol = inputs(g)
        if len(items) == 2:                           # same token count as the first question: batched with it
            gen = torch.Generator().manual_seed(99)
            image, crops = torch.randn(1, 3, 224, 224, generator=gen), torch.randn(2, 3, 224, 224, generator=gen)
            opts = [torch.randint(3, cfg.vocab - 24, (n,), generator=gen) for n in (6, 1, 3)]
        items.append((q[0].tolist(), [o.tolist() for o in opts], image.half().cuda(), crops.half().cuda(), il, ol))
    single = [eng.option_losses_batch([it])[0] for it in items]
    batch = eng.option_losses_batch(items)
    for (l1, c1), (lb, cb) in zip(single, batch):
        assert float((lb - l1).abs().max()) < 5e-3, (l1, lb)
    assert torch.equal(batch[1][0], single[1][0])


def test_device_pixels_f16_equal_host_half(setup):
    """VQA_LLM.device_pixels on an fp16 engine == the host path's fp32 pixels .half(), bit for bit"""
    from PIL import Image
    from vstar_b200 import seal
    from vstar_b200.image import GpuImagePipeline
    from vstar_b200.vqa import VQA_LLM, _clip_preprocess
    V, O, cfg, sd, eng = setup

    class Src:
        def __init__(self):
            self.pipeline = GpuImagePipeline("cuda", 224, 768)

        def resident(self, im):
            return self.pipeline.upload(im)

    vqa, host = VQA_LLM(engine=eng), VQA_LLM(engine=eng)
    vqa.use_device_images(Src())
    for k, (w, h) in enumerate([(640, 640), (900, 500), (333, 777)]):
        img = Image.fromarray(np.random.default_rng(60 + k).integers(0, 256, (h, w, 3), dtype=np.uint8), "RGB")
        boxes = [[w * 0.3, h * 0.4, w * 0.1, h * 0.12], [2.0, 3.0, 500.0, 600.0]]
        img_d, crops_d = vqa.device_pixels(img, boxes, patch_scale=1.2)
        bg = tuple(int(x * 255) for x in host.image_processor.image_mean)
        padded, _, _ = seal.expand2square_center(img, bg)
        img_h = _clip_preprocess(padded).unsqueeze(0).half().cuda()
        crops_h = torch.stack([host.get_object_crop(img, b, patch_scale=1.2) for b in boxes], 0).half().cuda()
        torch.cuda.synchronize()
        assert img_d.dtype == F16 and torch.equal(img_d, img_h), (w, h, float((img_d.float() - img_h.float()).abs().max()))
        assert torch.equal(crops_d, crops_h), (w, h)
        a, b = host._pixels(padded, torch.stack([host.get_object_crop(img, b, patch_scale=1.2) for b in boxes], 0))
        assert torch.equal(a, img_h) and torch.equal(b, crops_h)


def test_model_adapter_half_inputs(setup):
    """LlavaSearchModel (what load_pretrained_model(..., torch_dtype=torch.float16) returns) driven like vstar_bench_eval.py with
    .half() pixels: forward with images, forward per option on past_key_values, generate"""
    from vstar_b200.vqa import VQA_LLM
    V, O, cfg, sd, eng = setup
    model = VQA_LLM(engine=eng).model
    rng = np.random.default_rng(11)
    gen = torch.Generator().manual_seed(3)
    image, crops = torch.randn(1, 3, 224, 224, generator=gen).half(), torch.randn(2, 3, 224, 224, generator=gen).half()
    q = [1] + rng.integers(3, cfg.vocab - 30, 6).tolist() + [-200] + rng.integers(3, cfg.vocab - 30, 5).tolist() + [-300] + \
        rng.integers(3, cfg.vocab - 30, 3).tolist() + [-300] + rng.integers(3, cfg.vocab - 30, 4).tolist()
    opts = [rng.integers(3, cfg.vocab - 30, n).tolist() for n in (3, 5, 2)]
    il, ol = [False], [True, False]
    qt = torch.tensor([q])
    out_q = model(qt, use_cache=True, images=image, object_features=crops, images_long=il, objects_long=ol)
    T = 32 + 256 + 32 + (len(q) - 3)
    assert out_q.logits.shape == (1, T, cfg.vocab)
    losses = []
    for opt in opts:
        ot = torch.tensor([opt])
        o = model(input_ids=ot.cuda(), use_cache=True, past_key_values=out_q.past_key_values)
        logits = torch.cat([out_q.logits[:, -1:], o.logits[:, :-1]], 1)
        losses.append(torch.nn.CrossEntropyLoss()(logits.view(-1, cfg.vocab).float(), ot.view(-1).cuda()))
    losses = torch.stack(losses).cpu()
    ref_losses, choice = eng.option_losses(q, opts, image.cuda(), crops.cuda(), il, ol)
    assert torch.allclose(losses, ref_losses, rtol=2e-3, atol=2e-3) and int(losses.argmin()) == choice
    model.eos_token_id = -1
    out = model.generate(qt, images=image, object_features=crops, images_long=il, objects_long=ol, do_sample=False, max_new_tokens=3)
    assert out.shape == (1, len(q) + 3) and out[0, :len(q)].tolist() == q
    assert out[0, len(q):].tolist() == eng.generate(q, image.cuda(), crops.cuda(), il, ol, max_new_tokens=3, eos_token_id=-1)


def test_vqa_fp16_from_streamed_checkpoint(setup, tmp_path):
    """an fp16 safetensors checkpoint streamed through open_checkpoint into VQAWeights(..., dtype=torch.float16) equals
    from_state_dict(..., dtype=torch.float16)"""
    from safetensors.torch import save_file
    from vstar_b200.checkpoint import open_checkpoint
    from vstar_b200.vqa import VQAWeights
    V, O, cfg, sd, eng = setup
    d = tmp_path / "vqa"
    os.makedirs(d)
    main = {k: v.half().contiguous() for k, v in sd.items()}
    keys = sorted(main)
    save_file({k: main[k] for k in keys[::2]}, str(d / "model-00001-of-00002.safetensors"))
    save_file({k: main[k] for k in keys[1::2]}, str(d / "model-00002-of-00002.safetensors"))
    w = VQAWeights(cfg, open_checkpoint(str(d), device="cuda"), dtype=F16)
    ref = eng.w
    torch.cuda.synchronize()
    for a, b in zip(w.layers, ref.layers):
        for k in a:
            assert a[k].dtype == F16 and torch.equal(a[k], b[k]), k
    for name in ("lm_head", "embed", "final_norm", "rope_cos", "mm_w", "latents", "media_pos"):
        assert torch.equal(getattr(w, name), getattr(ref, name)), name
    assert torch.equal(w.clip["patch_w"], ref.clip["patch_w"]) and torch.equal(w.pj_layers[3]["wkv"], ref.pj_layers[3]["wkv"])


def test_seal_answer_fp16_vqa_with_bf16_vsm(setup):
    """one seal_answer with the fp16 VQA LLM and the bf16 VSM in the same process"""
    from PIL import Image
    from oracle import vsm_oracle as O2
    from vstar_b200.engine import VSMEngine, VSMWeights
    from vstar_b200.seal import MISSING_OBJECTS_MSG, seal_answer
    from vstar_b200.vqa import VQA_LLM
    from vstar_b200.vsm import VSM
    V, O, cfg, sd, eng = setup
    vsd = O2.synthetic_state_dict(cfg, seed=1234)
    prompt, ans = O2.synthetic_prompt(cfg, n_text=24, seed=5)

    class V2(VSM):
        def _ids(self, q):
            return prompt[0].tolist()

    vsm = V2(engine=VSMEngine(VSMWeights.from_state_dict(cfg, vsd)), forced_answer_ids=ans.tolist(), frontier_batch=8)
    assert vsm.engine.dtype == BF
    vqa = VQA_LLM(engine=eng)
    img = Image.fromarray(np.random.default_rng(9).integers(0, 256, (480, 700, 3), dtype=np.uint8), "RGB")
    res = seal_answer(vqa, vsm, img, "What colour is the mug?", ["red", "blue", "green", "white"],
                      prediction_override=MISSING_OBJECTS_MSG + " mug, laptop.",
                      search_kwargs=dict(confidence_high=2.0, target_cue_threshold=-1e9, target_cue_threshold_minimum=-1e9))
    assert res["missing_objects"] == ["mug", "laptop"] and len(res["search_result"]) == 2
    assert res["option_chosen"] in (0, 1, 2, 3)
