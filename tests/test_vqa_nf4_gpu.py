"""The SEAL VQA LLM in its 4-bit mode (NF4 weights, fp16 compute; the reference's load_4bit) on the NF4 kernels.

(1) format: the CUDA quantiser's codes, absmax and scales are bit-identical to oracle/nf4_oracle.py, the dequantiser to the
    oracle's dequantisation (random tensors at Llama-7B shapes and edge blocks);
(2) GEMM: vsb_gemm_nf4 against fp32 x @ deq(W)^T with every variant forced, every epilogue and the row remap; criterion
    err <= 2 * err(torch fp16 matmul on deq(W)) + ATOL; the dequant + tile path is bit-identical to vsb_gemm_f16 on deq(W);
(3) the native layer runner on an NF4 table == the same kernels sequenced from Python, bit for bit (prefill, ragged decode, option pass);
(4) the NF4 engine against vqa_oracle in fp32 on the dequantised state dict (the reference's 4-bit math) on the goldens;
(5) the rest of the VQA surface on the NF4 engine, and the memory footprint of the load."""
import json
import os

import numpy as np
import pytest
import torch

from tests.helpers import REPORT_DIR

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
BF, F16 = torch.bfloat16, torch.float16
ATOL = 2e-3


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


def tuned(force_bn):
    from vstar_b200 import _lib

    class Ctx:
        def __enter__(self):
            _lib.call("vsb_gemm_set_tuning", force_bn, 0)

        def __exit__(self, *a):
            _lib.call("vsb_gemm_set_tuning", 0, 0)
    return Ctx()


def _oracle_equal(ops, w):
    from oracle import nf4_oracle as N
    q = ops.nf4_quantize(w)
    absmax = torch.empty((w.shape[0], w.shape[1] // 64), dtype=torch.float32, device="cuda")
    codes = torch.empty_like(q.codes)
    ops.call("vsb_nf4_quantize", w.data_ptr(), w.shape[0], w.shape[1], codes.data_ptr(), absmax.data_ptr(), ops._stream())
    offset = float(absmax.mean())
    c_ref, a_ref, s_ref = N.quantize(w.cpu(), offset=offset)
    torch.cuda.synchronize()
    assert torch.equal(q.codes.cpu(), torch.from_numpy(c_ref))
    assert torch.equal(absmax.cpu(), torch.from_numpy(a_ref))
    assert torch.equal(q.scales.cpu(), torch.from_numpy(s_ref))
    deq = ops.nf4_dequant(q)
    assert torch.equal(deq.cpu(), torch.from_numpy(N.dequantize(c_ref, s_ref)))
    return q, deq


# ------------------------------------------------------------------------------------------------ (1) format
@pytest.mark.parametrize("N_,K", [(4096, 4096), (11008, 4096), (4096, 11008), (3, 320)])
def test_quantizer_and_dequantizer_equal_the_oracle(ops, N_, K):
    if K % 64:
        with pytest.raises(ops._lib.VsbError):
            ops.nf4_quantize(rnd(N_, K))
        return
    _oracle_equal(ops, rnd(N_, K, scale=0.02, seed=K))


def test_edge_blocks(ops):
    w = torch.randn(8, 256).mul(0.05).half()
    w[0] = 0                                               # all-zero row: zeros whatever the scale
    w[1, :64] = 0
    w[1, 17] = 0.3                                         # a single non-zero value
    w[2, :64] = torch.tensor([0.25, -0.25] * 32)           # exactly +-absmax
    w[3, :] = torch.tensor([6e-8, -1.2e-7, 3e-6, 5.9e-5]).half().repeat(64)     # fp16 subnormals
    q, deq = _oracle_equal(ops, w.cuda())
    deq = deq.cpu()
    assert torch.equal(deq[0], torch.zeros(256, dtype=F16))
    assert deq[1, 17] != 0 and torch.equal(deq[1, :17], torch.zeros(17, dtype=F16))
    codes = q.codes.cpu()
    assert torch.all(codes[2, :32] == 0xF0)                # +absmax -> code 15, -absmax -> code 0
    zeros = torch.zeros(4, 128, dtype=F16, device="cuda")
    qz, dz = _oracle_equal(ops, zeros)
    assert torch.equal(dz, zeros) and torch.all(qz.codes == 0x77)


# ------------------------------------------------------------------------------------------------ (2) GEMM
def _gemm_case(ops, M, N_, K, epi, force, seed=0):
    a = rnd(M, K, seed=1 + seed)
    q = ops.nf4_quantize(rnd(N_, K, scale=K ** -0.5, seed=2 + seed))
    wd = ops.nf4_dequant(q)
    b, r = rnd(N_, scale=0.1, seed=3), rnd(M, N_, seed=4)
    kw = {}
    if "bias" in epi:
        kw["bias"] = b
    if "res" in epi:
        kw["residual"] = r
    if epi == "fp32":
        kw["out_dtype"] = torch.float32
        if "res" in epi:
            kw["residual"] = r.float()
    code = dict(quick_gelu=ops.EPI_QUICK_GELU, gelu=ops.EPI_GELU, swiglu=ops.EPI_SWIGLU, relu=ops.EPI_RELU).get(epi, ops.EPI_NONE)
    with tuned(force):
        out = ops.gemm(a, q, epilogue=code, **kw)
        dense = ops.gemm(a, wd, epilogue=code, **kw) if force not in (1, 2) else None
    torch.cuda.synchronize()

    def ref(dt):
        y = a.to(dt) @ wd.to(dt).t()
        if "bias" in kw:
            y = y + b.to(dt)
        if code == ops.EPI_QUICK_GELU:
            y = y * torch.sigmoid(1.702 * y)
        elif code == ops.EPI_GELU:
            y = torch.nn.functional.gelu(y)
        elif code == ops.EPI_RELU:
            y = torch.relu(y)
        elif code == ops.EPI_SWIGLU:
            y = torch.nn.functional.silu(y[:, 0::2]) * y[:, 1::2]
        if "residual" in kw:
            y = y + r.to(dt)
        return y
    e, et = err(out, ref(torch.float32)), err(ref(F16), ref(torch.float32))
    assert e <= 2 * et + ATOL, (M, N_, K, epi, force, e, et)
    if dense is not None and (force != 0 or M > 32):
        assert torch.equal(out, dense), (M, N_, K, epi, force)      # dequant + tile path == vsb_gemm_f16 on deq(W)
    return e


SHAPES_7B = [(12288, 4096, "none"), (4096, 11008, "res"), (22016, 4096, "swiglu"), (4096, 4096, "fp32")]
SHAPES_TINY = [(768, 256, "bias"), (1024, 256, "swiglu"), (256, 512, "res"), (1024, 1024, "quick_gelu"), (320, 128, "gelu"),
               (256, 256, "relu")]


@pytest.mark.parametrize("M", [1, 2, 5, 8, 16, 17, 64, 600])
def test_gemm_nf4_auto(ops, M):
    for N_, K, epi in SHAPES_7B + SHAPES_TINY:
        _gemm_case(ops, M, N_, K, epi, 0)


@pytest.mark.parametrize("force", [1, 2, 64, 128, 256])
def test_gemm_nf4_forced_variants(ops, force):
    Ms = [1, 2, 5, 8] if force == 1 else [1, 5, 8, 16, 17, 24, 32] if force == 2 else [1, 17, 64, 600]
    for M in Ms:
        for N_, K, epi in SHAPES_7B[:3] + SHAPES_TINY[:3]:
            _gemm_case(ops, M, N_, K, epi, force)
    with tuned(force), pytest.raises(ops._lib.VsbError):
        if force in (1, 2):
            ops.gemm(rnd(40, 256), ops.nf4_quantize(rnd(64, 256)))
        else:
            raise ops._lib.VsbError("tile widths take any M")


def test_gemm_nf4_row_remap(ops):
    """rows scattered through rows_per_group (5 groups, 3 rows of gap between them) land where vsb_gemm_f16 puts them on the
    dequantised weight, with every variant"""
    K = 1024
    q = ops.nf4_quantize(rnd(1024, K, scale=K ** -0.5, seed=5))
    wd = ops.nf4_dequant(q)
    for M, force in ((5, 1), (10, 2), (40, 0), (600, 128)):
        a = rnd(M, K, seed=6)
        rpg = M // 5
        kw = dict(rows_per_group=rpg, group_stride=rpg + 3, group_offset=2)
        out = torch.zeros((5 * (rpg + 3) + 2, 1024), dtype=F16, device="cuda")
        with tuned(force):
            ops.gemm(a, q, out=out, **kw)
        ref = torch.zeros_like(out)
        with tuned(0 if force in (1, 2) else force):
            ops.gemm(a, wd, out=ref, **kw)
        torch.cuda.synchronize()
        assert err(out, ref) < 2e-3 and torch.equal(out == 0, ref == 0)
    with pytest.raises(ops._lib.VsbError):
        ops.gemm(rnd(4, 96), ops.NF4Weight(torch.zeros((8, 48), dtype=torch.uint8, device="cuda"),
                                           torch.zeros((8, 1), device="cuda"), 8, 96))


# ------------------------------------------------------------------------------------------------ (3) native runner
def _rope_tables(maxpos, D, theta=10000.0):
    inv = 1.0 / (theta ** (torch.arange(0, D, 2, dtype=torch.float32) / D))
    fr = torch.outer(torch.arange(maxpos, dtype=torch.float32), inv)
    return fr.cos().to(F16).cuda().contiguous(), fr.sin().to(F16).cuda().contiguous()


@pytest.mark.parametrize("d,H,inter", [(256, 2, 512), (1024, 8, 2048)])
def test_llama_layers_nf4_native_runner(ops, d, H, inter):
    """vsb_llama_layers_f16 on an NF4 table == the same kernels from Python, bit for bit: prefill Tn = 70, a ragged decode step
    (k_start), an option pass (q_seg); head_dim 128 takes the fused-RoPE QKV GEMM on the prefill.  The bf16 entry point and a
    table that mixes NF4 and dense projections are refused."""
    nl, B, Tmax = 2, 2, 128
    hd = d // H
    layers = [dict(ln1=(1 + 0.1 * torch.randn(d)).to(F16).cuda(), wqkv=ops.nf4_quantize(rnd(3 * d, d, scale=d ** -0.5, seed=70 + i)),
                   wo=ops.nf4_quantize(rnd(d, d, scale=d ** -0.5, seed=80 + i)), ln2=(1 + 0.1 * torch.randn(d)).to(F16).cuda(),
                   wgu=ops.nf4_quantize(rnd(2 * inter, d, scale=d ** -0.5, seed=90 + i)),
                   wdown=ops.nf4_quantize(rnd(d, inter, scale=inter ** -0.5, seed=100 + i))) for i in range(nl)]
    cos_t, sin_t = _rope_tables(Tmax, hd)
    table = ops.llama_layer_table(layers)
    deq = torch.empty(2 * inter * d, dtype=F16, device="cuda")

    def python_stack(x, cache, Tn, past, positions=None, k_start=None, q_seg=None):
        ld = 3 * d
        rows = B * Tn
        attn = torch.empty((rows, d), dtype=F16, device="cuda")
        for li, L in enumerate(layers):
            h = ops.rmsnorm(x, L["ln1"], 1e-6)
            cl = cache[li].view(B * Tmax, ld)
            if hd == 128 and k_start is None and rows > 32:
                w = ops.nf4_dequant(L["wqkv"])
                ops.call("vsb_gemm_qkv_rope_f16", h.data_ptr(), d, w.data_ptr(), d, cl.data_ptr(), ld, rows, 3 * d, d, Tn, Tmax, past, 0, 0,
                         1e-6, rows, cos_t.data_ptr(), sin_t.data_ptr(), ops._p(positions), Tn, past, hd, ops._stream())
            else:
                ops.gemm(h, L["wqkv"], out=cl, rows_per_group=Tn, group_stride=Tmax, group_offset=past)
                ops.rope_(cl, Tn, H, hd, cos_t, sin_t, pos0=past, positions=positions, rows=rows, group_stride=Tmax, group_offset=past)
            args = (cl[past:], cl[:, d:], cl[:, 2 * d:], attn)
            strides = (Tmax * ld, ld, Tmax * ld, ld, Tmax * ld, ld, Tn * d, d)
            if q_seg is not None:
                ops.call("vsb_flash_attn_seg_f16", *[t.data_ptr() for t in args], *strides, B, H, Tn, past + Tn, hd, hd ** -0.5,
                         q_seg.data_ptr(), past, ops._stream())
            elif k_start is not None:
                ops.call("vsb_attn_decode_f16", *[t.data_ptr() for t in args], *strides, B, H, Tn, past + Tn, hd, 1, hd ** -0.5,
                         k_start.data_ptr(), ops._stream())
            else:
                ops.flash_attn(*args, B, H, Tn, past + Tn, hd, True, hd ** -0.5, *strides)
            ops.gemm(attn, L["wo"], out=x, residual=x)
            h = ops.rmsnorm(x, L["ln2"], 1e-6)
            gu = ops.gemm(h, L["wgu"], epilogue=ops.EPI_SWIGLU)
            ops.gemm(gu, L["wdown"], out=x, residual=x)
        return x

    def native_stack(x, cache, Tn, past, positions=None, k_start=None, q_seg=None):
        scratch = torch.empty(B * Tn * (2 * d + inter), dtype=F16, device="cuda")
        return ops.llama_layers(table, nl, x, B, Tn, past, cache, B, Tmax, d, H, inter, 1e-6, cos_t, sin_t, scratch, positions=positions,
                                k_start=k_start, q_seg=q_seg, seg_lo=past if q_seg is not None else 0, deq_scratch=deq)

    pos_dec = torch.tensor([70, 65], dtype=torch.int32, device="cuda")
    k_start = torch.tensor([0, 5], dtype=torch.int32, device="cuda")
    seg = torch.tensor([71, 71, 71, 74, 74, 74, 74, 74] * B, dtype=torch.int32, device="cuda")[:B * 8]
    pos_opt = torch.tensor([71, 72, 73, 71, 72, 73, 74, 75] * B, dtype=torch.int32, device="cuda")[:B * 8]
    outs = []
    for fn in (python_stack, native_stack):
        cache = torch.zeros(nl, B, Tmax, 3 * d, dtype=F16, device="cuda")
        y0 = fn(rnd(B * 70, d, seed=110).clone(), cache, 70, 0).clone()
        y1 = fn(rnd(B, d, seed=111).clone(), cache, 1, 70, positions=pos_dec, k_start=k_start).clone()
        y2 = fn(rnd(B * 8, d, seed=112).clone(), cache, 8, 71, positions=pos_opt, q_seg=seg).clone()
        outs.append((y0, y1, y2, cache.clone()))
    torch.cuda.synchronize()
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)
    assert torch.isfinite(outs[0][0].float()).all() and float(outs[0][0].float().abs().max()) > 0
    with pytest.raises(Exception):
        ops.llama_layer_table([dict(layers[0]), dict(layers[1], wo=ops.nf4_dequant(layers[1]["wo"]))])

    def raw_call(fn, tab):
        x, cache = rnd(B, d, seed=113).clone(), torch.zeros(nl, B, Tmax, 3 * d, dtype=F16, device="cuda")
        scratch = torch.empty(B * (2 * d + inter), dtype=F16, device="cuda")
        ops.call(fn, tab, nl, x.data_ptr(), B, 1, 0, cache.data_ptr(), B, Tmax, d, H, inter, 1e-6, cos_t.data_ptr(), sin_t.data_ptr(),
                 None, None, 0, None, 0, 0, scratch.data_ptr(), deq.data_ptr(), ops._stream())

    with pytest.raises(ops._lib.VsbError):
        raw_call("vsb_llama_layers", table)
    mixed = (type(table[0]) * nl)(*table)
    mixed[1].wo_scales = None
    with pytest.raises(ops._lib.VsbError):
        raw_call("vsb_llama_layers_f16", mixed)


# ------------------------------------------------------------------------------------------------ (4) engine parity
@pytest.fixture(scope="module")
def setup():
    from oracle import nf4_oracle as N, vqa_oracle as V, vsm_oracle as O
    from vstar_b200 import synth
    from vstar_b200.vqa import VQAEngine, VQAWeights
    cfg = O.tiny_config()
    sd = {k: synth.synthetic_tensor(k, shp, seed=4321) for k, shp in V.vqa_state_dict_shapes(cfg).items()}
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    eng = VQAEngine(VQAWeights.from_state_dict(cfg, sd, dtype=F16, quant="nf4"), max_tokens=1024)
    peak = torch.cuda.max_memory_allocated() - base
    sdq = N.dequantized_state_dict(sd)
    return V, O, cfg, sd, sdq, eng, peak


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


@pytest.mark.parametrize("sub", ["short_long", "long_short"])
def test_nf4_engine_parity_on_goldens(setup, sub):
    V, O, cfg, sd, sdq, eng, _ = setup
    from vstar_b200.ops import NF4Weight
    assert isinstance(eng.w.layers[0]["wqkv"], NF4Weight) and isinstance(eng.w.pj_out[0], NF4Weight) and eng.w.quant == "nf4"
    g = np.load(os.path.join(G, f"vqa_a_{sub}.npz"))
    image, crops, q, opts, il, ol = inputs(g)
    e32 = V.build_embeds(sdq, cfg, q, image, crops, il, ol)
    l32 = V.forward_logits(sdq, cfg, e32)
    sd16 = {k: v.half() for k, v in sdq.items()}
    l16 = V.forward_logits(sd16, cfg, V.build_embeds(sd16, cfg, q, image.half(), crops.half(), il, ol))
    e_oracle16 = err(l16[0], l32[0])
    ref_l, _ = V.option_losses(sdq, cfg, q, opts, image, crops, il, ol)
    ic, cc = image.half().cuda(), crops.half().cuda()
    x = eng.build_embeds(q[0].tolist(), ic, cc, il, ol)
    T = x.shape[0]
    eng.prefill_embeds(x)
    _, am, logits = eng._logits_rows(x, torch.arange(T, device="cuda"))
    e4 = err(logits, l32[0])
    assert e4 <= 2 * e_oracle16 + 1e-3, (e4, e_oracle16)
    losses, choice = eng.option_losses(q[0].tolist(), [o.tolist() for o in opts], ic, cc, il, ol)
    nll = float((losses - ref_l).abs().max())
    assert nll < 2e-3, (losses, ref_l)
    srt = ref_l.sort().values
    if float(srt[1] - srt[0]) > 2 * 2e-3:
        assert choice == int(ref_l.argmin())
    top2 = l32[0].topk(2, dim=-1).values
    confident = (top2[:, 0] - top2[:, 1]) > 1e-2
    assert torch.equal(am.cpu().long()[confident], l32[0].argmax(-1)[confident])
    l_unq = V.forward_logits(sd, cfg, V.build_embeds(sd, cfg, q, image, crops, il, ol))
    json.dump(dict(nf4=dict(logits_err=e4, nll_err=nll, losses=losses.tolist(), choice=choice), fp16_oracle_logits_err=e_oracle16,
                   ref_losses=ref_l.tolist(), info_distance_to_unquantized_reference=dict(logits=err(l32[0], l_unq[0]))),
              open(os.path.join(REPORT_DIR, f"vqa_nf4_parity_{sub}.json"), "w"), indent=1)


# ------------------------------------------------------------------------------------------------ (5) surface and memory
def rel(a, b):
    return err(torch.as_tensor(a).cpu(), torch.as_tensor(b).cpu())


def test_nf4_batched_decode_and_options(setup):
    V, O, cfg, sd, sdq, eng, _ = setup
    rng = np.random.default_rng(5)
    gen = torch.Generator().manual_seed(7)
    reqs = []
    for n_pre, n_post, long_ in ((5, 9, True), (12, 30, False), (3, 4, True)):
        ids = [1] + rng.integers(3, cfg.vocab - 30, n_pre).tolist() + [-200] + rng.integers(3, cfg.vocab - 30, n_post).tolist()
        reqs.append((ids, torch.randn(1, 3, 224, 224, generator=gen).half().cuda(), None, [long_], None))
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
    batch_rows = [logits.clone()]
    for s_ in range(3):
        batch_rows.append(eng.decode_ragged([f[s_] for f in forced], lens, Tpad, s_).clone())
    for b in range(3):
        got = torch.stack([r[b] for r in batch_rows])
        assert rel(got, single[b]) < 3e-2, (b, rel(got, single[b]))
    outs = eng.generate_batch(reqs, max_new_tokens=4, eos_token_id=-1)
    assert [len(o) for o in outs] == [4, 4, 4]
    items = []
    for sub in ("short_long", "long_short"):
        g = np.load(os.path.join(G, f"vqa_a_{sub}.npz"))
        image, crops, q, opts, il, ol = inputs(g)
        items.append((q[0].tolist(), [o.tolist() for o in opts], image.half().cuda(), crops.half().cuda(), il, ol))
    single = [eng.option_losses_batch([it])[0] for it in items]
    batch = eng.option_losses_batch(items)
    for (l1, c1), (lb, cb) in zip(single, batch):
        assert float((lb - l1).abs().max()) < 5e-3, (l1, lb)


def test_nf4_vqa_llm_and_model_adapter(setup):
    from vstar_b200.vqa import VQA_LLM
    V, O, cfg, sd, sdq, eng, _ = setup
    vqa = VQA_LLM(engine=eng)
    model = vqa.model
    rng = np.random.default_rng(11)
    gen = torch.Generator().manual_seed(3)
    image, crops = torch.randn(1, 3, 224, 224, generator=gen).half(), torch.randn(2, 3, 224, 224, generator=gen).half()
    q = [1] + rng.integers(3, cfg.vocab - 30, 6).tolist() + [-200] + rng.integers(3, cfg.vocab - 30, 5).tolist() + [-300] + \
        rng.integers(3, cfg.vocab - 30, 3).tolist() + [-300] + rng.integers(3, cfg.vocab - 30, 4).tolist()
    opts = [rng.integers(3, cfg.vocab - 30, n).tolist() for n in (3, 5, 2)]
    il, ol = [False], [True, False]
    qt = torch.tensor([q])
    out_q = model(qt, use_cache=True, images=image, object_features=crops, images_long=il, objects_long=ol)
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
    assert out[0, len(q):].tolist() == eng.generate(q, image.cuda(), crops.cuda(), il, ol, max_new_tokens=3, eos_token_id=-1)
    from PIL import Image
    img = Image.fromarray(np.random.default_rng(9).integers(0, 256, (300, 400, 3), dtype=np.uint8), "RGB")
    a = vqa.free_form_inference(img, "What is it?", max_new_tokens=3)
    b = vqa.free_form_inference_batch([img, img], ["What is it?", "What is it?"], max_new_tokens=3)
    assert isinstance(a, str) and b[0] == b[1]
    r = vqa.multiple_choices_inference(img, "What colour?", ["red", "blue"])
    rb = vqa.multiple_choices_inference_batch([(img, "What colour?", ["red", "blue"], None, None, None)])
    assert r is not None and rb[0] in (0, 1)


def test_nf4_memory_footprint(setup):
    """weight bytes of the quantised Linears = the formula from the shapes; the load's peak stays within the NF4 footprint plus the
    largest fp16 tensor plus a margin"""
    V, O, cfg, sd, sdq, eng, peak = setup
    from oracle import nf4_oracle as N
    shapes = V.vqa_state_dict_shapes(cfg)
    qk = N.quantized_keys(shapes)
    n = sum(int(np.prod(shapes[k])) for k in qk)
    assert eng.w.linear_bytes() == n // 2 + n // 64 * 4
    dense = sum(int(np.prod(s)) * 2 for k, s in shapes.items() if k not in qk)
    largest = max(int(np.prod(shapes[k])) * 2 for k in shapes)
    margin = 8 << 20                                      # RoPE tables, fused-layout copies of one layer, allocator rounding
    assert peak <= n // 2 + n // 64 * 4 + dense + largest + margin, (peak, n, dense, largest)


def test_load_pretrained_model_4bit_and_seal_answer(setup, tmp_path):
    """load_pretrained_model(load_4bit=True) on a tiny safetensors checkpoint == VQAWeights(..., quant="nf4") from the state dict;
    then one seal_answer with the NF4 VQA LLM next to the bf16 VSM"""
    from safetensors.torch import save_file
    from vstar_b200.checkpoint import open_checkpoint
    from vstar_b200.vqa import VQAWeights
    V, O, cfg, sd, sdq, eng, _ = setup
    d = tmp_path / "vqa"
    os.makedirs(d)
    save_file({k: v.half().contiguous() for k, v in sd.items()}, str(d / "model.safetensors"))
    w = VQAWeights(cfg, open_checkpoint(str(d), device="cuda"), dtype=F16, quant="nf4")
    torch.cuda.synchronize()
    for a, b in zip(w.layers, eng.w.layers):
        for k in ("wqkv", "wo", "wgu", "wdown"):
            assert torch.equal(a[k].codes, b[k].codes) and torch.equal(a[k].scales, b[k].scales), k
        assert torch.equal(a["ln1"], b["ln1"])
    assert torch.equal(w.pj_layers[2]["wkv"].codes, eng.w.pj_layers[2]["wkv"].codes) and torch.equal(w.lm_head, eng.w.lm_head)
    try:
        import transformers  # noqa: F401
        from vstar_b200 import vqa as vqa_mod
        import vstar_b200.vsm as vsm_mod
        orig = vsm_mod.config_from_hf
        vsm_mod.config_from_hf = lambda p: cfg

        class Tok:
            eos_token_id = 2

        import transformers as tr
        orig_tok = tr.AutoTokenizer.from_pretrained
        tr.AutoTokenizer.from_pretrained = staticmethod(lambda *a, **k: Tok())
        try:
            tok, model, proc, ctx = vqa_mod.load_pretrained_model(str(d), load_4bit=True)
        finally:
            vsm_mod.config_from_hf = orig
            tr.AutoTokenizer.from_pretrained = orig_tok
        assert model.engine.dtype == F16 and model.engine.w.quant == "nf4"
        assert torch.equal(model.engine.w.layers[1]["wgu"].codes, eng.w.layers[1]["wgu"].codes)
    except ImportError:
        pass
    from PIL import Image
    from oracle import vsm_oracle as O2
    from vstar_b200.engine import VSMEngine, VSMWeights
    from vstar_b200.seal import MISSING_OBJECTS_MSG, seal_answer
    from vstar_b200.vqa import VQA_LLM
    from vstar_b200.vsm import VSM
    vsd = O2.synthetic_state_dict(cfg, seed=1234)
    prompt, ans = O2.synthetic_prompt(cfg, n_text=24, seed=5)

    class V2(VSM):
        def _ids(self, q):
            return prompt[0].tolist()

    vsm = V2(engine=VSMEngine(VSMWeights.from_state_dict(cfg, vsd)), forced_answer_ids=ans.tolist(), frontier_batch=8)
    img = Image.fromarray(np.random.default_rng(9).integers(0, 256, (480, 700, 3), dtype=np.uint8), "RGB")
    res = seal_answer(VQA_LLM(engine=eng), vsm, img, "What colour is the mug?", ["red", "blue", "green", "white"],
                      prediction_override=MISSING_OBJECTS_MSG + " mug, laptop.",
                      search_kwargs=dict(confidence_high=2.0, target_cue_threshold=-1e9, target_cue_threshold_minimum=-1e9))
    assert res["missing_objects"] == ["mug", "laptop"] and res["option_chosen"] in (0, 1, 2, 3)
