"""Slot decode (VQAEngine.decode_stream): a decode batch whose rows sit at their own cache slot and length, so a request is
admitted whenever another one ends.

(1) vsb_rope_scatter == the row written to its cache row and rotated there by ops.rope_, bit for bit;
(2) vsb_attn_decode_slots == vsb_attn_decode_* (k_start NULL) bit for bit for equal lengths and slot[b] = b, and against a
    float64 reference at ragged lengths on permuted, non-contiguous slots;
(3) the stream on the bf16, fp16 and NF4 engines: in batch-invariant mode a request's logits do not depend on when it was
    admitted, next to whom or in which slot; in default mode they follow the fp32 oracle; the engine's own cache and the
    stream do not disturb each other; refusals raise before any launch; close() returns the device memory;
(4) answer_open_many == answer_open per item, with searches equal to the same searches run alone."""
import gc
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
BF, F16 = torch.bfloat16, torch.float16
SFX = {BF: "bf16", F16: "f16"}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ops():
    from vstar_b200 import ops as o
    return o


def randn(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def rope_tables(maxpos, hd, dt):
    inv = 1.0 / (10000.0 ** (torch.arange(0, hd, 2, dtype=torch.float32) / hd))
    fr = torch.outer(torch.arange(maxpos, dtype=torch.float32), inv)
    return fr.cos().to(dt).cuda(), fr.sin().to(dt).cuda()


def bits(t):
    return t.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("dt", [BF, F16])
@pytest.mark.parametrize("H,D", [(4, 128), (6, 64)])
def test_rope_scatter_equals_rope_in_place(ops, dt, H, D):
    Bc, Tmax, B = 12, 96, 9
    W = 3 * H * D
    g = torch.Generator().manual_seed(H * D)
    slot = torch.randperm(Bc, generator=g)[:B].to(torch.int32)
    length = torch.randint(0, Tmax, (B,), generator=g, dtype=torch.int32)
    pos = torch.randint(0, 2048, (B,), generator=g, dtype=torch.int32)
    cos, sin = rope_tables(2048, D, dt)
    qkv = randn(B, W + 24, seed=1).to(dt).cuda()[:, :W]                   # strided rows
    cache = randn(Bc, Tmax, W, seed=2).to(dt).cuda()
    ref = cache.clone()
    flat = ref.view(Bc * Tmax, W)
    for b in range(B):
        r = int(slot[b]) * Tmax + int(length[b])
        flat[r] = qkv[b]
        ops.rope_(flat[r:r + 1], 1, H, D, cos, sin, positions=pos[b:b + 1].cuda().contiguous())
    ops.rope_scatter(qkv, cache, H, D, cos, sin, slot.cuda(), length.cuda(), pos.cuda())
    torch.cuda.synchronize()
    assert torch.equal(bits(cache), bits(ref))


def slot_attn_ref(cache, slot, length, H, D, scale):
    """float64: row b's query at cache[slot[b], length[b], :HD] against keys / values [0, length[b]] of its slot"""
    c = cache.double()
    HD = H * D
    out = []
    for s, n in zip(slot.tolist(), length.tolist()):
        q = c[s, n, :HD].view(H, D)
        k = c[s, :n + 1, HD:2 * HD].view(n + 1, H, D)
        v = c[s, :n + 1, 2 * HD:].view(n + 1, H, D)
        p = torch.softmax(torch.einsum("hd,khd->hk", q, k) * scale, -1)
        out.append(torch.einsum("hk,khd->hd", p, v).reshape(HD))
    return torch.stack(out)


@pytest.mark.parametrize("dt", [BF, F16])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("B,Sk", [(1, 1), (3, 64), (5, 65), (32, 700), (64, 300), (8, 2047)])
def test_attn_slots_equal_decode_kernel_when_aligned(ops, dt, D, B, Sk):
    """equal lengths, slot[b] = b: bit-identical to vsb_attn_decode_* with Sq = 1 and k_start NULL"""
    H = 4
    HD, W, Tmax = H * D, 3 * H * D, Sk + 8
    cache = randn(B, Tmax, W, seed=B + Sk).to(dt).cuda()
    slot = torch.arange(B, dtype=torch.int32, device="cuda")
    length = torch.full((B,), Sk - 1, dtype=torch.int32, device="cuda")
    got = torch.empty((B, HD), dtype=dt, device="cuda")
    ops.attn_decode_slots(cache, got, H, D, D ** -0.5, slot, length)
    ref = torch.empty((B, HD), dtype=dt, device="cuda")
    base = cache.data_ptr()
    ops.call(f"vsb_attn_decode_{SFX[dt]}", base + (Sk - 1) * W * 2, base + HD * 2, base + 2 * HD * 2, ref.data_ptr(), Tmax * W, W,
             Tmax * W, W, Tmax * W, W, HD, HD, B, H, 1, Sk, D, 1, D ** -0.5, None, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert torch.equal(bits(got), bits(ref))


@pytest.mark.parametrize("dt", [BF, F16])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("keys", [[1], [2], [63], [64], [65], [2047], [1, 2, 63, 64, 65, 2047, 300, 1000],
                                  [1 + (37 * i) % 900 for i in range(64)]])
def test_attn_slots_ragged_against_float64(ops, dt, D, keys):
    """ragged key counts on permuted, non-contiguous slots (the slots in between hold NaN); batch-invariant mode gives every
    row the value it has alone"""
    H, Tmax = 2, 2048
    B = len(keys)
    Bc = 2 * B + 1
    W = 3 * H * D
    g = torch.Generator().manual_seed(B * D)
    slot = (torch.randperm(B, generator=g) * 2 + 1).to(torch.int32)
    length = torch.tensor([k - 1 for k in keys], dtype=torch.int32)
    cache = torch.full((Bc, Tmax, W), float("nan"), dtype=dt)
    vals = randn(B, Tmax, W, seed=D + B).to(dt)
    for b in range(B):
        cache[int(slot[b]), :keys[b]] = vals[b, :keys[b]]
    cache = cache.cuda()
    ref = slot_attn_ref(cache.cpu(), slot, length, H, D, D ** -0.5)
    out = torch.empty((B, H * D), dtype=dt, device="cuda")
    ops.attn_decode_slots(cache, out, H, D, D ** -0.5, slot.cuda(), length.cuda(), max_len=2047)
    torch.cuda.synchronize()
    ulp = 2.0 ** -8 if dt == BF else 2.0 ** -11
    err = (out.double().cpu() - ref).abs()
    assert bool((err <= 2 * ulp * ref.abs() + 4 * ulp * ref.abs().max()).all()), float(err.max())
    from vstar_b200 import ops as o
    with o.batch_invariant():
        full = torch.empty_like(out)
        o.attn_decode_slots(cache, full, H, D, D ** -0.5, slot.cuda(), length.cuda())
        for b in (0, B - 1):
            one = torch.empty((1, H * D), dtype=dt, device="cuda")
            o.attn_decode_slots(cache, one, H, D, D ** -0.5, slot[b:b + 1].cuda(), length[b:b + 1].cuda())
            assert torch.equal(bits(one[0]), bits(full[b]))


# ------------------------------------------------------------------------------------------------ engine
@pytest.fixture(scope="module")
def model():
    from oracle import vqa_oracle as V, vsm_oracle as O
    from vstar_b200 import synth
    cfg = O.tiny_config()
    sd = {k: synth.synthetic_tensor(k, shp, seed=4321) for k, shp in V.vqa_state_dict_shapes(cfg).items()}
    return V, cfg, sd


_ENGINES = {}


def engine(model, kind):
    from vstar_b200.vqa import VQAEngine, VQAWeights
    if kind not in _ENGINES:
        V, cfg, sd = model
        kw = dict(bf16={}, fp16=dict(dtype=F16), nf4=dict(dtype=F16, quant="nf4"))[kind]
        _ENGINES[kind] = VQAEngine(VQAWeights.from_state_dict(cfg, sd, **kw), max_tokens=1024)
    return _ENGINES[kind]


def requests(cfg, dtype, n, seed=5):
    rng = np.random.default_rng(seed)
    gen = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        ids = [1] + rng.integers(3, cfg.vocab - 30, 3 + 4 * i).tolist() + [-200] + rng.integers(3, cfg.vocab - 30, 5 + 3 * i).tolist()
        image = torch.randn(1, 3, 224, 224, generator=gen)
        out.append((ids, image.to(dtype).cuda(), None, [i % 2 == 0], None))
    return out


def run_target(eng, target, fillers, admit_at, steps, budgets):
    """stream of 4 slots: the fillers are admitted at step 0 with `budgets`, the target at step `admit_at` -> (target's logits
    rows, its tokens, its slot)"""
    rows = []
    st = eng.decode_stream(4, max_positions=512, eos_token_id=-1)
    try:
        for f, n in zip(fillers, budgets):
            st.admit(f, n)
        for _ in range(admit_at):
            st.step()
        h = st.admit(target, steps + 1)
        rows.append(st.last_logits[1][0].clone())
        for _ in range(steps):
            st.step()
            reqs, logits = st.last_logits
            rows.append(logits[[r.id for r in reqs].index(h.id)].clone())
        return torch.stack(rows), list(h.tokens), h.slot
    finally:
        st.close()


@pytest.mark.parametrize("kind", ["bf16", "fp16", "nf4"])
def test_stream_logits_do_not_depend_on_admission(model, ops, kind):
    V, cfg, sd = model
    eng = engine(model, kind)
    reqs = requests(cfg, eng.dtype, 4)
    target, fillers = reqs[0], reqs[1:]
    with ops.batch_invariant():
        alone, toks, slot0 = run_target(eng, target, [], 0, 6, [])
        slots = {slot0}
        for s in (0, 1, 7, 50):
            got, toks2, slot = run_target(eng, target, fillers, s, 6, [3, 70, 70])
            slots.add(slot)
            assert torch.equal(got, alone), (kind, s)
            assert toks2 == toks
    assert len(slots) >= 2                       # other slot indices, and a retired filler's slot reused (s = 7, 50)


def test_stream_follows_the_oracle(model, ops):
    """default mode: per-step logits within the decode tolerance of the fp32 oracle along each request's own path, and every
    emitted token a (near-)argmax; 3 requests on 2 slots, so the third is admitted when the first ends"""
    V, cfg, sd = model
    eng = engine(model, "bf16")
    reqs = requests(cfg, BF, 3, seed=9)
    budgets = [3, 6, 4]
    rows = {}
    st = eng.decode_stream(2, max_positions=400, eos_token_id=-1)
    handles = {}
    pending = list(range(3))

    def admit():
        i = pending.pop(0)
        h = st.admit(reqs[i], budgets[i])
        handles[h.id] = i
        rows.setdefault(i, []).append(st.last_logits[1][0].clone())

    admit()
    admit()
    finished = {}
    while len(finished) < 3:
        done = st.step()
        rs, logits = st.last_logits
        for k, r in enumerate(rs):
            rows[handles[r.id]].append(logits[k].clone())
        for r, toks in done:
            finished[handles[r.id]] = toks
        while pending and st.free_slots:
            admit()
    st.close()
    emb = sd["model.embed_tokens.weight"]
    for i, (ids, img, _, il, _) in enumerate(reqs):
        toks = finished[i]
        assert len(toks) == budgets[i]
        e = V.build_embeds(sd, cfg, torch.tensor([ids]), img.float().cpu(), None, il, None)
        for s_, t in enumerate(toks):
            ref = V.forward_logits(sd, cfg, e)[0, -1]
            got = rows[i][s_].cpu()
            assert float((got - ref).abs().max() / ref.abs().max()) < 3e-2, (i, s_)
            assert float(ref.max() - ref[t]) < 3e-2
            e = torch.cat([e, emb[torch.tensor([t])].unsqueeze(0)], dim=1)


def test_stream_and_engine_cache_do_not_disturb_each_other(model, ops):
    V, cfg, sd = model
    eng = engine(model, "bf16")
    reqs = requests(cfg, BF, 3, seed=11)
    rng = np.random.default_rng(3)
    q = [1] + rng.integers(3, 200, 6).tolist() + [-200] + rng.integers(3, 200, 8).tolist()
    opts = [rng.integers(3, 200, n).tolist() for n in (3, 5)]
    before = eng.option_losses(q, opts, reqs[0][1])[0]
    epoch = eng.kv_epoch

    def run(interrupt):
        st = eng.decode_stream(3, max_positions=400, eos_token_id=-1)
        for r in reqs:
            st.admit(r, 8)
        out = []
        for k in range(7):
            st.step()
            out.append(st.last_logits[1].clone())
            if interrupt and k == 2:
                during = eng.option_losses(q, opts, reqs[0][1])[0]
                assert torch.equal(during, before)
                eng.generate(reqs[1][0], reqs[1][1], max_new_tokens=3)
        st.close()
        return out

    plain = run(False)
    assert eng.kv_epoch == epoch
    mixed = run(True)
    assert all(torch.equal(a, b) for a, b in zip(plain, mixed))


def test_stream_refusals_raise_before_any_launch(model, ops):
    from vstar_b200 import _lib
    from vstar_b200.vqa import VQA_LLM
    V, cfg, sd = model
    eng = engine(model, "bf16")
    reqs = requests(cfg, BF, 2)
    with pytest.raises(NotImplementedError, match="temperature"):
        eng.decode_stream(2, temperature=0.7)
    with pytest.raises(NotImplementedError, match="num_beams"):
        eng.decode_stream(2, num_beams=2)
    with pytest.raises(_lib.VsbError):
        eng.decode_stream(2, max_positions=4096)
    st = eng.decode_stream(1, max_positions=300, eos_token_id=-1)
    T = eng.spliced_length(reqs[0][0], 0, reqs[0][3])
    n0 = _lib.launches
    with pytest.raises(_lib.VsbError, match="exceeds"):
        st.admit(reqs[0], 300 - T + 1)
    assert _lib.launches == n0
    st.admit(reqs[0], 5)
    n0 = _lib.launches
    with pytest.raises(RuntimeError, match="no free slot"):
        st.admit(reqs[1], 5)
    assert _lib.launches == n0
    st.close()
    # the refusals pinned for the other generation paths are unchanged
    llm = VQA_LLM(engine=eng)
    with pytest.raises(NotImplementedError):
        llm.model.generate(torch.tensor([[1, -200, 5]]), images=reqs[0][1], do_sample=True)


def test_stream_close_returns_device_memory(model, ops):
    V, cfg, sd = model
    eng = engine(model, "fp16")
    reqs = requests(cfg, F16, 2)
    eng.decode_stream(1, max_positions=64).close()               # builds the layer table once
    gc.collect()
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    st = eng.decode_stream(2, max_positions=512, eos_token_id=-1)
    assert torch.cuda.memory_allocated() > m0
    for r in reqs:
        st.admit(r, 4)
    while st.active:
        st.step()
    st.close()
    del st
    gc.collect()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == m0


def test_free_form_inference_stream_equals_free_form_inference(model, ops):
    """every answer of the stream (admitted as slots free) == free_form_inference of that item alone, in batch-invariant mode"""
    from vstar_b200.vqa import VQA_LLM
    V, cfg, sd = model
    eng = engine(model, "bf16")
    llm = VQA_LLM(engine=eng)
    rng = np.random.default_rng(4)
    from PIL import Image
    items = []
    for i in range(5):
        img = Image.fromarray(rng.integers(0, 256, (60 + 10 * i, 80, 3), dtype=np.uint8), "RGB")
        items.append((img, " ".join(["word"] * (1 + i)), None, None, None))
    with ops.batch_invariant():
        got = dict(llm.free_form_inference_stream(items, max_new_tokens=6, slots=2))
        want = {i: llm.free_form_inference(it[0], it[1], max_new_tokens=6) for i, it in enumerate(items)}
    assert got == want


# ------------------------------------------------------------------------------------------------ pipeline
def test_answer_open_many_equals_answer_open(model, ops):
    from oracle import vsm_oracle as O
    from PIL import Image
    from vstar_b200 import seal
    from vstar_b200.engine import VSMEngine, VSMWeights
    from vstar_b200.visual_search import visual_search
    from vstar_b200.vqa import VQA_LLM
    from vstar_b200.vsm import VSM
    V, cfg, sd = model
    j = json.load(open(os.path.join(ROOT, "tests", "golden", "tiny_config.json")))
    vcfg = O.VSMConfig(**j["cfg"])
    vsm_eng = VSMEngine(VSMWeights.from_state_dict(vcfg, O.synthetic_state_dict(vcfg, seed=j["weight_seed"])))
    prompt, ans = O.synthetic_prompt(vcfg, n_text=24, seed=11)
    from tests.helpers import FakeNLP
    from vstar_b200 import noun_chunks
    noun_chunks.set_nlp(FakeNLP())                # the weak-cue branch's noun chunker (spaCy is not a test dependency)

    class TinyVSM(VSM):
        def _ids(self, question):
            return prompt[0].tolist()

    vsm = TinyVSM(engine=vsm_eng, forced_answer_ids=ans.tolist(), frontier_batch=4)
    missing = {0: ["mug", "cup"], 2: ["dog"], 3: ["a", "b", "c"]}

    class ScriptedLLM(VQA_LLM):
        """the direct answers name scripted missing objects (random weights never do); final answers are the model's own"""

        def free_form_inference_stream(self, items, max_new_tokens=200, slots=16):
            for i, text in super().free_form_inference_stream(items, max_new_tokens=max_new_tokens, slots=slots):
                q = items[i][1]
                if seal.FOCUS_MSG not in q and int(q.split()[-1]) in missing:
                    text = seal.MISSING_OBJECTS_MSG + " " + ", ".join(missing[int(q.split()[-1])]) + "."
                yield i, text

    llm = ScriptedLLM(engine=engine(model, "bf16"))
    rng = np.random.default_rng(8)
    items = [(Image.fromarray(rng.integers(0, 256, (200 + 30 * i, 260, 3), dtype=np.uint8), "RGB"), f"what is in image {i}")
             for i in range(4)]
    # no detection is confident (random weights would find hundreds of boxes): each search walks its tree and keeps its best
    # fallback box, one object crop per missing object
    kw = dict(minimum_size=128, search_batch=4, search_kwargs=dict(confidence_high=2.0))
    with ops.batch_invariant():
        many = seal.answer_open_many(llm, vsm, items, slots=2, searches_in_flight=3, **kw)
        one = [seal.answer_open(llm, vsm, im, q, **kw) for im, q in items]
    assert many[1][1:] == (None, None, None) and one[1][1:] == (None, None, None)
    for a, b in zip(many, one):
        assert a[0] == b[0] and a[1] == b[1] and a[3] == b[3]
        assert (a[2] is None and b[2] is None) or np.array_equal(a[2], b[2])
    # the searches of the batched run == the same searches alone
    for i, names in missing.items():
        image = items[i][0]
        smallest = seal.smallest_size_for(image, 4.0, 128)
        alone = [visual_search(vsm, image, n, None, smallest, confidence_high=2.0, confidence_low=0.3, batch_size=4) for n in names]
        _, summary, annotated = seal.open_final_request(llm, image, items[i][1], names, alone)
        assert many[i][0] == seal.NEED_SEARCH_MSG.format(", ".join(names))
        assert many[i][1] == summary and np.array_equal(many[i][2], annotated)
    noun_chunks.set_nlp(None)
