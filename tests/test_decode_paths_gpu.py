"""The SEAL VQA LLM's decode and answer-option paths against plain float64 references, at the edges where kernels go wrong.

(1) Attention: vsb_attn_decode_* with per-sequence k_start (ragged decode), vsb_flash_attn_seg_* (answer options appended back
    to back after a cached prefix) and the causal diagonal of the prefill kernels.  Random inputs alone hide boundary errors (a
    leaked or dropped key moves a softmax over hundreds of random keys by less than the tolerance), so every case also sets
    probes: a masked key aimed at its query (scaled score ~ +30) with V = 8 (a leak moves the output by O(1)), the first and
    last visible key aimed at some queries (dropping one moves it by O(1)), and NaN in the cache rows that must never be read.
    Criterion: err(kernel) <= 2 * err(float64 softmax with P rounded to the operand dtype before P.V) + ATOL, errors max |x - ref|
    per (row, head) over that head's max |ref|.
(2) The native layer runner in its ragged-prefill / ragged-decode / option modes: == the same kernels sequenced from Python, bit
    for bit, and within 3e-2 of a float64 Llama stack that runs every sequence and every option alone (HF RMSNorm, rotate-half
    RoPE at the true positions, SwiGLU on the interleaved gate / up rows).  This catches a convention that the runner and the
    Python sequence share (a position off by one, what k_start means, where a segment starts).
(3) Token heads: argmax_rows (torch.argmax's order, NaN included), nll_rows (float64 logsumexp - x[label]) and the few-row
    RMSNorm kernel of the 7B decode shape.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
BF, F16 = torch.bfloat16, torch.float16
DTYPES = [BF, F16]
SFX = {BF: "bf16", F16: "f16"}
ATOL = {BF: 8e-3, F16: 2e-3}          # output rounding: 2^-9 (bf16) / 2^-12 (fp16) of a value, plus fp32 accumulation
NAN = float("nan")
PROBE_SCORE, LEAK_V = 30.0, 8.0


@pytest.fixture(scope="module")
def ops():
    from vstar_b200 import ops as o
    return o


def randn(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


# ------------------------------------------------------------------------------------------------ attention references
def attn_ref(q, k, v, mask, scale, dt):
    """q [Sq, H, D], k / v [Sk, H, D] (values of dtype dt), mask bool [Sq, Sk] (True = visible) ->
    (float64 attention, the same with P rounded to dt before P.V), both [Sq, H, D] float64"""
    q, k, v = (t.double().transpose(0, 1) for t in (q, k, v))
    s = (q @ k.transpose(1, 2)) * scale
    p = torch.softmax(s.masked_fill(~mask.to(s.device), float("-inf")), -1)
    return (p @ v).transpose(0, 1), (p.to(dt).double() @ v).transpose(0, 1)


def head_err(a, ref):
    """max over (row, head) of max |a - ref| / max(max |ref|, 0.05) within the head; NaN anywhere -> inf"""
    a, ref = a.double(), ref.double()
    if not torch.isfinite(a).all():
        return math.inf
    return float(((a - ref).abs().amax(-1) / ref.abs().amax(-1).clamp_min(0.05)).max())


def check_attn(got, r64, rlo, dt, what):
    e, et = head_err(got, r64), head_err(rlo, r64)
    assert e <= 2 * et + ATOL[dt], (what, e, et)


class Probes:
    """aims keys of a float32 K [B, S, H, D] at queries q [B, Sq, H, D] (a key is aimed at one query per head at most)"""

    def __init__(self, q, k, v, scale):
        self.q, self.k, self.v, self.scale, self.used = q, k, v, scale, set()

    def aim(self, b, h, qrow, key, leak=False):
        h %= self.k.shape[2]
        if (b, h, key) in self.used:
            return
        self.used.add((b, h, key))
        qv = self.q[b, qrow, h].float()
        self.k[b, key, h] = qv * (PROBE_SCORE / (self.scale * float(qv.pow(2).sum())))
        if leak:
            self.v[b, key, h] = LEAK_V


# ------------------------------------------------------------------------------------------------ (1) ragged decode
def decode_cluster(B, H, Sk, sms):
    """cluster size launch_decode (csrc/attention.cu) picks: keys of a (batch, head) split over 8, 4, 2 or 1 CTAs"""
    s = 8
    while s > 1 and (s * H * B > 2 * sms + H or Sk // s < 64):
        s //= 2
    return s


@pytest.mark.parametrize("dt", DTYPES, ids=["bf16", "f16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("B,H,Sk,cluster", [(1, 32, 600, 8), (2, 3, 383, 4), (2, 4, 130, 2), (8, 32, 600, 1)])
def test_ragged_decode(ops, dt, D, B, H, Sk, cluster):
    """vsb_attn_decode_* with k_start against each sequence alone on its unpadded keys: Sq 1, 2, 4 (4 takes the NQ = 4
    template), every cluster size, k_start 0, 1, Sk - Sq and 3 visible keys over 8 splits (trailing splits empty), on a strided
    cache whose rows before k_start and from Sk on hold NaN"""
    assert decode_cluster(B, H, Sk, torch.cuda.get_device_properties(0).multi_processor_count) == cluster
    Tmax, scale = Sk + 40, D ** -0.5
    for Sq in (1, 2, 4):
        off = Sk - Sq
        starts = [0, 1, off, Sk - max(Sq, 3), 63, Sk // 2, 5, off - 1]
        for L in range(max(1, 4 // B)):
            ks = [starts[(L * B + b) % len(starts)] for b in range(B)]
            seed = 1000 * Sq + 10 * L + D
            q = randn(B, Sq, H, D, seed=seed).to(dt)
            k, v = randn(B, Tmax, H, D, seed=seed + 1), randn(B, Tmax, H, D, seed=seed + 2)
            pr = Probes(q, k, v, scale)
            for b in range(B):
                if Sq > 1:
                    pr.aim(b, 0, 0, off + 1, leak=True)               # beyond query 0's causal diagonal
                pr.aim(b, 1, Sq - 1, ks[b])                           # first visible key
                for qi in range(Sq):
                    pr.aim(b, 2, qi, off + qi)                        # each query's diagonal key
            kc, vc = k.to(dt), v.to(dt)
            for t in (kc, vc):
                t[:, Sk:] = NAN
                for b in range(B):
                    t[b, :ks[b]] = NAN
            qd, kd, vd = q.cuda(), kc.cuda(), vc.cuda()
            out = torch.full((B, Sq, H, D), NAN, dtype=dt, device="cuda")
            k_start = torch.tensor(ks, dtype=torch.int32, device="cuda")
            HD = H * D
            ops.call(f"vsb_attn_decode_{SFX[dt]}", qd.data_ptr(), kd.data_ptr(), vd.data_ptr(), out.data_ptr(), Sq * HD, HD, Tmax * HD, HD,
                     Tmax * HD, HD, Sq * HD, HD, B, H, Sq, Sk, D, 1, scale, k_start.data_ptr(), ops._stream())
            torch.cuda.synchronize()
            for b in range(B):
                n = Sk - ks[b]
                mask = torch.ones(Sq, n, dtype=torch.bool).tril(n - Sq)
                r64, rlo = attn_ref(qd[b], kd[b, ks[b]:Sk], vd[b, ks[b]:Sk], mask, scale, dt)
                check_attn(out[b], r64, rlo, dt, ("decode", Sq, b, ks[b]))


# ------------------------------------------------------------------------------------------------ (1) option segments
SEG_LAYOUTS = [[40, 30, 70], [1, 64, 5], [63, 2, 17, 1]]     # option lengths of batch entries 0, 1, 2 (140 rows: 3 query tiles)


@pytest.mark.parametrize("dt", DTYPES, ids=["bf16", "f16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("seg_lo", [0, 1, 63, 64, 600])
def test_segment_mask(ops, dt, D, seg_lo):
    """vsb_flash_attn_seg_*: options appended back to back after a prefix of seg_lo rows, right-padded as VQAEngine's option
    scoring pads them (a padding row's segment starts at the row itself), Q a strided view of the fused q|k|v cache, O rows
    wider than H*D; each option (and each padding row) against the prefix alone plus its own rows"""
    P, scale = seg_lo, D ** -0.5
    for B, H in ((1, 32), (3, 2)):
        layouts = SEG_LAYOUTS[:B]
        Sq = max(sum(lens) for lens in layouts)
        Sk, Tmax, HD = P + Sq, P + Sq + 24, H * D
        c = randn(B, Tmax, 3, H, D, seed=7 * D + P + B)
        q = c[:, P:P + Sq, 0].to(dt)
        pr = Probes(q, c[:, :, 1], c[:, :, 2], scale)
        seg = torch.zeros(B, Sq, dtype=torch.int32)
        spans = []                                           # (b, first row, rows) of every option and padding row
        for b, lens in enumerate(layouts):
            s = 0
            for n in lens:
                seg[b, s:s + n] = P + s
                spans.append((b, s, n))
                s += n
            for r in range(s, Sq):
                seg[b, r] = P + r
                spans.append((b, r, 1))
        for b, s, n in spans:
            if s > 0:
                pr.aim(b, 0, s, P + s - 1, leak=True)            # head 0, leaks: last row of the previous option,
            if n > 1:
                pr.aim(b, 0, s, P + s + 1, leak=True)            # and the key beyond the causal diagonal
            pr.aim(b, 1, s + n - 1, P + s)                       # head 1, keeps: first row of its own option,
            pr.aim(b, 1, s, P + s + n - 1 if n > 1 else P + s)   # the diagonal,
            if P:
                pr.aim(b, 1, s, 0)                               # the first and last prefix keys
                pr.aim(b, 1, s + n - 1, P - 1)
        cache = c.to(dt)
        cache[:, Sk:] = NAN
        cd = cache.cuda().view(B * Tmax, 3 * HD)
        ld_o = HD + 64
        out = torch.full((B * Sq, ld_o), -7.0, dtype=dt, device="cuda")
        segd = seg.cuda().view(-1)
        ops.call(f"vsb_flash_attn_seg_{SFX[dt]}", cd[P:].data_ptr(), cd[:, HD:].data_ptr(), cd[:, 2 * HD:].data_ptr(), out.data_ptr(),
                 Tmax * 3 * HD, 3 * HD, Tmax * 3 * HD, 3 * HD, Tmax * 3 * HD, 3 * HD, Sq * ld_o, ld_o, B, H, Sq, Sk, D, scale,
                 segd.data_ptr(), P, ops._stream())
        torch.cuda.synchronize()
        assert bool((out[:, HD:] == -7.0).all())
        got = out[:, :HD].view(B, Sq, H, D)
        kv = cd.view(B, Tmax, 3, H, D)
        for b, s, n in spans:
            keys = torch.cat([torch.arange(P), torch.arange(P + s, P + s + n)]).cuda()
            mask = torch.cat([torch.ones(n, P, dtype=torch.bool), torch.ones(n, n, dtype=torch.bool).tril()], 1)
            r64, rlo = attn_ref(kv[b, P + s:P + s + n, 0], kv[b, keys, 1], kv[b, keys, 2], mask, scale, dt)
            check_attn(got[b, s:s + n], r64, rlo, dt, ("seg", B, H, b, s, n))


# ------------------------------------------------------------------------------------------------ (1) causal prefill diagonal
@pytest.mark.parametrize("dt", DTYPES, ids=["bf16", "f16"])
@pytest.mark.parametrize("impl", [1, 2, 3])
@pytest.mark.parametrize("D", [64, 128])
def test_causal_prefill_diagonal(ops, dt, impl, D):
    """the prefill kernels (1 = mma.sync, 2 = wgmma, 3 = wgmma with one query warpgroup per CTA) on Sq new rows after Sk - Sq
    cached ones (shared-prefix and chunked-prefill shapes), strided fused cache with NaN rows from Sk on"""
    from vstar_b200 import _lib
    B, H, scale = 2, 3, D ** -0.5
    HD = H * D
    _lib.call("vsb_attn_set_impl", impl)
    try:
        for Sq in (1, 63, 64, 65, 130):
            for off in (0, 1, 64, 300):
                Sk, Tmax = Sq + off, Sq + off + 16
                c = randn(B, Tmax, 3, H, D, seed=Sq * 7 + off + D)
                q = c[:, off:Sk, 0].to(dt)
                pr = Probes(q, c[:, :, 1], c[:, :, 2], scale)
                rows = sorted({0, Sq // 2, 62, 63, 64, Sq - 1} & set(range(Sq)))
                for b in range(B):
                    for qi in rows:
                        if qi + 1 < Sq:
                            pr.aim(b, 0, qi, off + qi + 1, leak=True)
                        pr.aim(b, 1, qi, off + qi)
                    pr.aim(b, 2, rows[-1 if b == 0 else len(rows) // 2], 0)
                cache = c.to(dt)
                cache[:, Sk:] = NAN
                cd = cache.cuda().view(B * Tmax, 3 * HD)
                out = torch.full((B * Sq, HD), NAN, dtype=dt, device="cuda")
                ops.flash_attn(cd[off:], cd[:, HD:], cd[:, 2 * HD:], out, B, H, Sq, Sk, D, True, scale, Tmax * 3 * HD, 3 * HD,
                               Tmax * 3 * HD, 3 * HD, Tmax * 3 * HD, 3 * HD, Sq * HD, HD)
                torch.cuda.synchronize()
                kv = cd.view(B, Tmax, 3, H, D)
                mask = torch.ones(Sq, Sk, dtype=torch.bool).tril(off)
                for b in range(B):
                    r64, rlo = attn_ref(kv[b, off:Sk, 0], kv[b, :Sk, 1], kv[b, :Sk, 2], mask, scale, dt)
                    check_attn(out.view(B, Sq, H, D)[b], r64, rlo, dt, ("prefill", impl, Sq, off, b))
    finally:
        _lib.call("vsb_attn_set_impl", 0)


# ------------------------------------------------------------------------------------------------ (2) layer runner modes
EPS = 1e-6


def rope_tables(maxpos, hd, dt):
    inv = 1.0 / (10000.0 ** (torch.arange(0, hd, 2, dtype=torch.float32) / hd))
    fr = torch.outer(torch.arange(maxpos, dtype=torch.float32), inv)
    return fr.cos().to(dt).cuda(), fr.sin().to(dt).cuda()


def python_stack(ops, layers, x, cache, B, Tn, past, H, cos_t, sin_t, row_off=0, positions=None, k_start=None, q_seg=None, seg_lo=0):
    """the layer sequence of csrc/llama_layers.cu (dense weights, unfolded norms) from Python, cache origin shifted by row_off rows"""
    sfx = SFX[x.dtype]
    d = x.shape[1]
    hd, ld, rows = d // H, 3 * d, B * Tn
    Bc, Tmax = cache.shape[1], cache.shape[2]
    attn = torch.empty((rows, d), dtype=x.dtype, device="cuda")
    for li, L in enumerate(layers):
        h = ops.rmsnorm(x, L["ln1"], EPS)
        cl = cache[li].view(Bc * Tmax, ld)[row_off:]
        if hd == 128 and d % 256 == 0 and k_start is None and rows > 16:      # the tile GEMMs take RoPE into their epilogue
            ops.call(f"vsb_gemm_qkv_rope_{sfx}", h.data_ptr(), d, L["wqkv"].data_ptr(), d, cl.data_ptr(), ld, rows, 3 * d, d, Tn, Tmax, past,
                     0, 0, EPS, rows, cos_t.data_ptr(), sin_t.data_ptr(), ops._p(positions), Tn, past, hd, ops._stream())
        else:
            ops.gemm(h, L["wqkv"], out=cl, rows_per_group=Tn, group_stride=Tmax, group_offset=past)
            ops.rope_(cl, Tn, H, hd, cos_t, sin_t, pos0=past, positions=positions, rows=rows, group_stride=Tmax, group_offset=past)
        ptrs = [t.data_ptr() for t in (cl[past:], cl[:, d:], cl[:, 2 * d:], attn)]
        strides = (Tmax * ld, ld, Tmax * ld, ld, Tmax * ld, ld, Tn * d, d)
        if q_seg is not None:
            ops.call(f"vsb_flash_attn_seg_{sfx}", *ptrs, *strides, B, H, Tn, past + Tn, hd, hd ** -0.5, q_seg.data_ptr(), seg_lo, ops._stream())
        elif k_start is not None:
            ops.call(f"vsb_attn_decode_{sfx}", *ptrs, *strides, B, H, Tn, past + Tn, hd, 1, hd ** -0.5, k_start.data_ptr(), ops._stream())
        else:
            ops.flash_attn(cl[past:], cl[:, d:], cl[:, 2 * d:], attn, B, H, Tn, past + Tn, hd, True, hd ** -0.5, *strides)
        ops.gemm(attn, L["wo"], out=x, residual=x)
        h = ops.rmsnorm(x, L["ln2"], EPS)
        gu = ops.gemm(h, L["wgu"], epilogue=ops.EPI_SWIGLU)
        ops.gemm(gu, L["wdown"], out=x, residual=x)
    return x


def stack64(W, x, pos, H, cos64, sin64):
    """float64 Llama decoder layers over ONE sequence x [n, d] at RoPE positions pos [n], causal among its n rows"""
    n, d = x.shape
    hd = d // H
    c = torch.cat([cos64[pos], cos64[pos]], -1)[:, None]
    s = torch.cat([sin64[pos], sin64[pos]], -1)[:, None]

    def rms(t, w):
        return w * (t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + EPS))

    def rot(t):
        return torch.cat([-t[..., hd // 2:], t[..., :hd // 2]], -1)
    for L in W:
        q, k, v = (rms(x, L["ln1"]) @ L["wqkv"].T).view(n, 3, H, hd).unbind(1)
        q, k = q * c + rot(q) * s, k * c + rot(k) * s
        a = attn_ref(q, k, v, torch.ones(n, n, dtype=torch.bool).tril(), hd ** -0.5, torch.float64)[0]
        x = x + a.reshape(n, d) @ L["wo"].T
        gu = rms(x, L["ln2"]) @ L["wgu"].T
        x = x + (torch.nn.functional.silu(gu[:, 0::2]) * gu[:, 1::2]) @ L["wdown"].T
    return x


def rel(a, ref):
    return float((a.double() - ref).abs().max() / ref.abs().max())


@pytest.mark.parametrize("dt", DTYPES, ids=["bf16", "f16"])
@pytest.mark.parametrize("d,H", [(256, 2), (1024, 8)])
def test_layer_runner_ragged_and_options(ops, dt, d, H):
    """vsb_llama_layers{,_f16} on a dense table (2 layers): a prefill_ragged-style setup (left-padded sequences of 9, 20, 20 and
    37 rows, the equal ones prefilled as one batch, pad rows NaN), two decode_ragged steps (positions / k_start), and one option
    pass (q_seg) after two prefixes of 30 rows; (a) == the kernels from Python bit for bit, (b) within 3e-2 of the float64
    stack on every sequence / option alone; the option pass's nll_rows per-option means against the float64 cross-entropy"""
    nl, inter, V, Tmax = 2, 2 * d, 320, 64
    g = torch.Generator().manual_seed(d + H)

    def w(*shape, scale=1.0):
        return (torch.randn(*shape, generator=g) * scale).to(dt).cuda()
    layers = [dict(ln1=w(d, scale=0.1) + 1, wqkv=w(3 * d, d, scale=d ** -0.5), wo=w(d, d, scale=d ** -0.5), ln2=w(d, scale=0.1) + 1,
                   wgu=w(2 * inter, d, scale=d ** -0.5), wdown=w(d, inter, scale=inter ** -0.5)) for _ in range(nl)]
    emb, final, lm_head = w(V, d), w(d, scale=0.1) + 1, w(V, d, scale=d ** -0.5)
    W64 = [{k: t.double() for k, t in L.items()} for L in layers]
    cos_t, sin_t = rope_tables(Tmax, d // H, dt)
    cos64, sin64 = cos_t.double(), sin_t.double()
    table = ops.llama_layer_table(layers)

    def native_stack(x, cache, B, Tn, past, row_off=0, **kw):
        scratch = torch.empty(B * Tn * (2 * d + inter), dtype=dt, device="cuda")
        return ops.llama_layers(table, nl, x, B, Tn, past, cache, cache.shape[1], Tmax, d, H, inter, EPS, cos_t, sin_t, scratch,
                                cache_row_offset=row_off, **kw)

    def python(x, cache, B, Tn, past, row_off=0, **kw):
        return python_stack(ops, layers, x, cache, B, Tn, past, H, cos_t, sin_t, row_off=row_off, **kw)

    def i32(v):
        return torch.tensor(v, dtype=torch.int32, device="cuda")

    # ---- ragged prefill + decode
    lens, steps = [9, 20, 20, 37], 2
    Bc, Tpad = len(lens), max(lens)
    ids = [torch.randint(V, (n + steps,), generator=g).cuda() for n in lens]

    def ragged(stack):
        cache = torch.full((nl, Bc, Tmax, 3 * d), NAN, dtype=dt, device="cuda")
        pre, b = [], 0
        while b < Bc:
            G = 1
            while b + G < Bc and lens[b + G] == lens[b]:
                G += 1
            T = lens[b]
            x = emb[torch.cat([ids[b + j][:T] for j in range(G)])]
            stack(x, cache, G, T, 0, row_off=b * Tmax + Tpad - T)
            pre += list(x.view(G, T, d))
            b += G
        dec = []
        for s in range(steps):
            x = emb[torch.stack([ids[b][lens[b] + s] for b in range(Bc)])]
            stack(x, cache, Bc, 1, Tpad + s, positions=i32([n + s for n in lens]), k_start=i32([Tpad - n for n in lens]))
            dec.append(x)
        return [t.clone() for t in pre] + dec + [cache]

    # ---- option pass: the prefixes prefilled as one batch, then every option of both in one q_seg pass
    Tq, Tn = 30, 12
    opts = [[[int(t) for t in torch.randint(V, (n,), generator=g)] for n in lens_] for lens_ in ([3, 5, 4], [2, 6])]
    q_ids = torch.randint(V, (2, Tq), generator=g).cuda()
    o_ids, pos, seg = torch.zeros(2, Tn, dtype=torch.int64), torch.zeros(2, Tn, dtype=torch.int32), torch.zeros(2, Tn, dtype=torch.int32)
    for b, oo in enumerate(opts):                # as VQAEngine.option_losses_batch lays them out
        off = 0
        for o in oo:
            for j, tok in enumerate(o):
                o_ids[b, off + j], pos[b, off + j], seg[b, off + j] = tok, Tq + j, Tq + off
            off += len(o)
        for r in range(off, Tn):
            pos[b, r], seg[b, r] = Tq, Tq + r

    def options(stack):
        cache = torch.full((nl, 2, Tmax, 3 * d), NAN, dtype=dt, device="cuda")
        x = emb[q_ids.view(-1)]
        stack(x, cache, 2, Tq, 0)
        xo = emb[o_ids.view(-1).cuda()]
        stack(xo, cache, 2, Tn, Tq, positions=pos.view(-1).cuda(), q_seg=seg.view(-1).cuda(), seg_lo=Tq)
        return [x.clone(), xo, cache]

    res_py = ragged(python) + options(python)
    res_nat = ragged(native_stack) + options(native_stack)
    torch.cuda.synchronize()
    for a, b in zip(res_py, res_nat):                                           # (a), bits (the caches hold NaN pad rows)
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))

    # (b) every sequence alone: prefill rows, then the decode rows
    pre, dec = res_nat[:Bc], res_nat[Bc:Bc + steps]
    for b, n in enumerate(lens):
        ref = stack64(W64, emb[ids[b]].double(), torch.arange(n + steps).cuda(), H, cos64, sin64)
        assert rel(pre[b], ref[:n]) < 3e-2, (b, rel(pre[b], ref[:n]))
        for s in range(steps):
            assert rel(dec[s][b], ref[n + s:n + s + 1]) < 3e-2, (b, s, rel(dec[s][b], ref[n + s:n + s + 1]))

    # (b) every option alone on its prefix, every padding row alone on its prefix (one token 0 at position Tq)
    xq, xo = res_nat[Bc + steps + 1], res_nat[Bc + steps + 2].view(2, Tn, d)

    def logits64(x):
        return (final.double() * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + EPS))) @ lm_head.double().T

    def logits(x):
        return ops.gemm(ops.rmsnorm(x.contiguous(), final, EPS), lm_head, out_dtype=torch.float32)
    for b, oo in enumerate(opts):
        pref = q_ids[b]
        off = 0
        ref = stack64(W64, emb[pref].double(), torch.arange(Tq).cuda(), H, cos64, sin64)
        assert rel(xq.view(2, Tq, d)[b], ref) < 3e-2, (b, rel(xq.view(2, Tq, d)[b], ref))
        for o in oo + [[0]] * (Tn - sum(len(o) for o in oo)):
            n = len(o)
            ref = stack64(W64, emb[torch.cat([pref, torch.tensor(o).cuda()])].double(), torch.arange(Tq + n).cuda(), H, cos64, sin64)
            assert rel(xo[b, off:off + n], ref[Tq:]) < 3e-2, (b, off, n, rel(xo[b, off:off + n], ref[Tq:]))
            if off < sum(len(o) for o in oo):
                # the option's loss: rows Tq-1 .. Tq+n-2 predict its tokens (CrossEntropyLoss of vstar_bench_eval.py)
                rows = logits(torch.cat([xq.view(2, Tq, d)[b, Tq - 1:], xo[b, off:off + n - 1]]))
                labels = torch.tensor(o, dtype=torch.int64, device="cuda")
                nll = ops.nll_rows(rows, labels)
                r = logits64(ref[Tq - 1:Tq + n - 1])
                ce64 = float((torch.logsumexp(r, -1) - r[torch.arange(n), labels]).mean())
                dl = float((rows.double() - r).abs().max())
                assert abs(float(nll.double().mean()) - ce64) <= 2 * dl + 1e-4, (b, off, float(nll.mean()), ce64, dl)
                r32 = rows.double()
                ref_nll = torch.logsumexp(r32, -1) - r32[torch.arange(n), labels]
                assert torch.allclose(nll.double(), ref_nll, rtol=1e-5, atol=1e-5)
            off += n


# ------------------------------------------------------------------------------------------------ (3) token heads
def first_max(row):
    """torch.argmax's index on a 1-D fp32 CPU row: the first NaN if there is one, else the first maximum"""
    nan = torch.isnan(row)
    return int(nan.nonzero()[0]) if bool(nan.any()) else int((row == row.max()).nonzero()[0])


def argmax_rows_cases(n, seed):
    """rows of length n: random, ties at the maximum (one thread, across lanes, across warps, at the last index), +-inf, NaN"""
    x = randn(1, n, seed=seed).repeat(24, 1)
    big = 50.0

    def put(r, idx, val=big):
        for i in idx:
            if not 0 <= i < n or len(set(idx)) != len(idx):
                return
        x[r, list(idx)] = val
    put(1, [5, 5 + 256])                      # same thread (stride 256)
    put(2, [3, 17])                           # lanes of one warp
    put(3, [40, 200])                         # warps 1 and 6
    put(4, [n - 1])                           # unique maximum at the last index
    put(5, [n - 257, n - 1])                  # the last index ties with an earlier one in the same thread
    put(6, [n - 2, n - 1])                    # ... in neighbouring lanes
    put(7, [n // 2], math.inf)
    put(8, [n - 1, 1], math.inf)
    x[9] = -math.inf
    x[10, ::3] = -math.inf
    put(11, [n // 3], NAN)
    x[12] = NAN
    put(13, [n - 1, n // 2], NAN)
    put(14, [0], math.inf)
    put(14, [n - 1], NAN)
    x[15] = 1.5
    x[16] = -math.inf
    put(16, [n - 1], -1e30)
    put(17, [n - 300, n - 40, n - 1])         # three ties, the last in another warp
    x[18] = -3.0
    put(18, [n - 1], NAN)
    x[19, :] = 0.0
    x[20] = randn(n, seed=seed + 1) * 1e-30
    x[21] = -randn(n, seed=seed + 2).abs()
    x[22] = torch.arange(n, dtype=torch.float32).flip(0)
    x[23] = torch.arange(n, dtype=torch.float32)
    return x


@pytest.mark.parametrize("n", [1, 255, 256, 257, 320, 32000, 32004])
def test_argmax_rows(ops, n):
    """vsb_argmax_rows_f32 == torch.argmax on every row (first maximum wins, NaN is the maximum), val == x[idx], on rows that are
    views into a wider buffer"""
    x = argmax_rows_cases(n, seed=n)
    R = x.shape[0]
    buf = torch.full((R, n + 19), 1e38)
    buf[:, 3:3 + n] = x
    xd = buf.cuda()[:, 3:3 + n]
    idx, val = ops.argmax_rows(xd)
    torch.cuda.synchronize()
    idx, val = idx.cpu().long(), val.cpu()
    for r in range(R):
        ref = first_max(x[r])
        assert ref == int(torch.argmax(x[r])), (n, r)
        assert int(idx[r]) == ref, (n, r, int(idx[r]), ref)
    assert torch.equal(val.isnan(), x[torch.arange(R), idx].isnan())
    same = ~val.isnan()
    assert torch.equal(val[same], x[torch.arange(R), idx][same])


@pytest.mark.parametrize("n", [320, 32000, 32004])
def test_nll_rows(ops, n):
    """vsb_nll_rows_f32 == float64 logsumexp(x) - x[label] on strided rows: offsets of +-1e4 (overflow without the max
    subtraction), -inf entries (a label on one gives +inf), labels 0 and n - 1, and 0 for labels outside [0, n)"""
    rows = []
    labels = []
    for k, (shift, ninf) in enumerate([(0, False), (1e4, False), (-1e4, False), (0, True), (1e4, True), (-1e4, True)]):
        for lab in (0, n - 1, n // 3, -1, n):
            r = randn(n, seed=n + 10 * k + lab % 7) * 3 + shift
            if ninf:
                r[1::5] = -math.inf
            rows.append(r)
            labels.append(lab)
    r = randn(n, seed=n + 99)
    r[7] = -math.inf
    rows.append(r)
    labels.append(7)
    x = torch.stack(rows)
    R = x.shape[0]
    buf = torch.zeros(R, n + 40)
    buf[:, 8:8 + n] = x
    got = ops.nll_rows(buf.cuda()[:, 8:8 + n], torch.tensor(labels, dtype=torch.int64).cuda())
    torch.cuda.synchronize()
    got = got.cpu().double()
    xd = x.double()
    lse = torch.logsumexp(xd, -1)
    for i, lab in enumerate(labels):
        if not 0 <= lab < n:
            assert float(got[i]) == 0.0, (i, lab)
            continue
        ref = float(lse[i] - xd[i, lab])
        if math.isinf(ref):
            assert float(got[i]) == ref, (i, float(got[i]))
            continue
        mx = float(x[i][torch.isfinite(x[i])].abs().max())
        tol = 1e-5 * (1 + abs(ref)) + 2.0 ** -22 * mx
        assert abs(float(got[i]) - ref) <= tol, (i, lab, float(got[i]), ref, tol)


@pytest.mark.parametrize("dt", DTYPES, ids=["bf16", "f16"])
@pytest.mark.parametrize("rows", [1, 8, 32])
@pytest.mark.parametrize("cols", [2048, 4096])
def test_rmsnorm_decode_rows(ops, dt, rows, cols):
    """the few-row RMSNorm kernel (rows <= 32, cols >= 2048: the 7B decode shape) against HF's LlamaRMSNorm in the operand dtype
    (fp32 statistics, normalised row rounded to the dtype, times the weight, rounded again), on strided rows"""
    ulp = 2.0 ** -8 if dt == BF else 2.0 ** -11            # half the relative spacing of the dtype's values at worst
    x = (randn(rows, cols + 64, seed=rows + cols) * 2).to(dt).cuda()[:, :cols]
    wt = (1 + 0.1 * randn(cols, seed=cols)).to(dt).cuda()
    out = torch.full((rows, cols + 32), NAN, dtype=dt, device="cuda")
    ops.rmsnorm(x, wt, EPS, out=out[:, :cols])
    torch.cuda.synchronize()
    assert out[:, cols:].isnan().all()
    y = out[:, :cols].double()
    xf = x.float()
    hs = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + EPS)).to(dt)
    ref = (wt.float() * hs.float()).to(dt).double()
    assert bool(((y - ref).abs() <= 4 * ulp * ref.abs()).all()), float((y - ref).abs().max())
    assert float((y == ref).double().mean()) > 0.99
    xd = x.double()
    r64 = wt.double() * xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + EPS)
    assert bool(((y - r64).abs() <= 3 * ulp * r64.abs() + 2.0 ** -23).all())     # + fp16's subnormal spacing
