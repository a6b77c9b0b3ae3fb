"""Sampled and beam-search requests on the decode stream (DecodeStream.admit(temperature=, num_beams=)).

(1) vsb_sample_rows_var_f32 == oracle/sampling_oracle.py row by row with every row's own temperature, top_k, top_p, seed and
    step (ties, -inf, all-equal and dominant rows; V 320 / 32000; 1 / 3 / 64 rows; both logit dtypes), and == vsb_sample_rows_f32
    token for token when the settings are uniform;
(2) vsb_copy_slot_rows_b16 == torch indexing bit for bit over random (src, dst, lo, hi) sets, == vsb_copy_cache_rows_b16 for one
    range, and every refusal returns VSB_ERR_ARG with the cache untouched;
(3) in batch-invariant mode a sampled request's and a beam request's (k = 2, 4) per-step logits, tokens and final ids do not
    depend on when it is admitted, on its slots (retired requests' slots reused) or on its neighbours (greedy, sampled, beam);
(4) replayed on the stream's own logits: sampled tokens == the sampling oracle, beam ids and score == oracle/beam_oracle.py,
    top_k = 1 == greedy;
(5) free_form_inference_stream(temperature, top_p) == free_form_inference of each item in order after the same seed (and
    num_beams likewise); a greedy-only stream issues the parent step's launches in the same order with bit-identical logits; a
    mixed step makes one device-to-host copy; close() returns the device memory."""
import gc

import numpy as np
import pytest
import torch

from oracle import beam_oracle as BO
from oracle import sampling_oracle as S

pytestmark = pytest.mark.gpu
BF, F16 = torch.bfloat16, torch.float16
MARGIN = 1e-6


@pytest.fixture(scope="module")
def ops():
    from vstar_b200 import ops as o
    return o


# ------------------------------------------------------------------------------------------------ per-row sampler
def edge_rows(n, B, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, n, generator=g) * 2.5
    if B >= 5:
        x[0] = 1.0                                                            # all equal
        kth = x[1].sort(descending=True).values[49]
        x[1, torch.randperm(n, generator=g)[:max(60, n // 10)]] = kth          # wide tie at the 50th value
        x[2, torch.randperm(n, generator=g)[:int(0.4 * n)]] = -float("inf")
        x[3, int(torch.randint(0, n, (1,), generator=g))] = 40.0              # one dominant token
        x[4, : n // 2] = x[4, n // 2:]                                        # every value twice
    seeds = torch.randint(-2 ** 63, 2 ** 63 - 1, (B,), generator=g, dtype=torch.int64)
    return x, seeds


def row_settings(n, B, seed):
    rng = np.random.default_rng(seed)
    T = rng.choice([0.2, 0.7, 1.0, 1.5], B).astype(np.float32)
    k = rng.choice([0, 1, 50, n], B).astype(np.int32)
    p = rng.choice([0.0, 0.9, 1.0], B).astype(np.float32)
    step = rng.integers(0, 500, B).astype(np.int32)
    return T, k, p, step


def sample_var(ops, x, T, k, p, dtype, seeds, steps):
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return ops.sample_rows_var(x.cuda(), d(T), d(k), d(p), dtype, seeds.cuda(), d(steps))


@pytest.mark.parametrize("n", [320, 32000])
@pytest.mark.parametrize("dtype", [BF, F16])
@pytest.mark.parametrize("B", [1, 3, 64])
def test_per_row_sampler_matches_oracle(ops, n, dtype, B):
    x, seeds = edge_rows(n, B, seed=n + B + (dtype == F16))
    total = loose = 0
    for rep in range(4):
        T, k, p, steps = row_settings(n, B, seed=rep * 100 + B)
        got = sample_var(ops, x, T, k, p, dtype, seeds, steps).cpu().numpy()
        for b in range(B):
            r = S.sample_row(x[b], float(T[b]), int(k[b]), float(p[b]), dtype, int(seeds[b]), int(steps[b]))
            if got[b] != r["token"]:
                assert r["margin"] < MARGIN, (b, T[b], k[b], p[b], got[b], r["token"], r["margin"])
                loose += 1
            total += 1
    assert loose <= max(2, total // 1000), (loose, total)


@pytest.mark.parametrize("n", [320, 32000])
@pytest.mark.parametrize("dtype", [BF, F16])
def test_per_row_sampler_equals_scalar_sampler_when_uniform(ops, n, dtype):
    B = 64
    x, seeds = edge_rows(n, B, seed=7 + n)
    for T, k, p, step in ((0.7, 50, 0.9, 3), (1.0, 0, 0.9, 11), (1.5, 50, 1.0, 0), (0.2, n, 0.0, 41), (1.0, 1, 1.0, 5)):
        want = ops.sample_rows(x.cuda(), T, k, p, dtype, seeds.cuda(), step)
        got = sample_var(ops, x, np.full(B, T, np.float32), np.full(B, k, np.int32), np.full(B, p, np.float32), dtype, seeds,
                         np.full(B, step, np.int32))
        assert torch.equal(got, want), (T, k, p)


# ------------------------------------------------------------------------------------------------ ranged row copy
def cache_tensor(L=3, Bc=10, Tm=40, W=48, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-30000, 30000, (L, Bc, Tm, W), generator=g, dtype=torch.int16).view(BF).cuda()


def test_ranged_copy_equals_torch(ops):
    rng = np.random.default_rng(1)
    for trial in range(30):
        Bc = int(rng.integers(2, 12))
        cache = cache_tensor(Bc=Bc, W=int(rng.choice([48, 50])), seed=trial)      # W = 50: the scalar (unaligned) path
        n = int(rng.integers(1, Bc // 2 + 1))
        perm = rng.permutation(Bc)
        src, dst = perm[:n], perm[n:2 * n]
        quads = []
        for s, d in zip(src, dst):
            lo = int(rng.integers(0, 40))
            quads.append((int(s), int(d), lo, int(rng.integers(lo, 41))))
        ref = cache.clone()
        for s, d, lo, hi in quads:
            ref[:, d, lo:hi] = cache[:, s, lo:hi]
        ops.copy_slot_rows(cache, quads)
        torch.cuda.synchronize()
        assert torch.equal(cache.view(torch.int16), ref.view(torch.int16)), quads


def test_ranged_copy_uniform_equals_copy_cache_rows(ops):
    a = cache_tensor(Bc=12, seed=5)
    b = a.clone()
    pairs = [(0, 5), (1, 7), (2, 3), (4, 11)]
    ops.copy_cache_rows(a, pairs, 6, 29)
    ops.copy_slot_rows(b, [(s, d, 6, 29) for s, d in pairs])
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_ranged_copy_refusals(ops):
    import ctypes
    from vstar_b200 import _lib
    cache = cache_tensor(Bc=8, seed=9)
    before = cache.clone()
    L, Bc, Tm, W = cache.shape
    lib = _lib.load()
    bad = [[(0, 5, 0, 4), (5, 6, 0, 4)],          # slot 5 both a source and a destination
           [(1, 1, 0, 4)],                        # a slot copied onto itself
           [(0, 5, 0, 4), (1, 5, 2, 6)],          # destination named twice
           [(0, 8, 0, 4)], [(-1, 3, 0, 4)],       # slots outside [0, slots)
           [(0, 3, 5, 4)],                        # lo > hi
           [(0, 3, 0, Tm + 1)]]                   # past the slot
    for quads in bad:
        arr = (ctypes.c_int * (4 * len(quads)))(*[v for q in quads for v in q])
        rc = lib.vsb_copy_slot_rows_b16(cache.data_ptr(), L, cache.stride(0), Bc, cache.stride(1), cache.stride(2), W, arr, len(quads),
                                        torch.cuda.current_stream().cuda_stream)
        assert rc == -1, quads                    # VSB_ERR_ARG
        with pytest.raises(_lib.VsbError):
            ops.copy_slot_rows(cache, quads)
    torch.cuda.synchronize()
    assert torch.equal(cache.view(torch.int16), before.view(torch.int16))


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


SAMPLED = dict(temperature=0.7, top_k=50, top_p=0.9, seed=123)


def run_target(eng, target, tkw, fillers, admit_at, steps, slots=8, eos=-1):
    """fillers (request, budget, admit keywords) admitted at step 0, the target at step `admit_at` with `tkw` -> (its logits rows
    per step, its beams before every step, its tokens, score, slots)"""
    st = eng.decode_stream(slots, max_positions=512, eos_token_id=eos)
    try:
        for f, n, kw in fillers:
            st.admit(f, n, **kw)
        for _ in range(admit_at):
            st.step()
        h = st.admit(target, steps + 1, **tkw)
        rows, beams = [st.last_logits[1].clone()], [[[]]]
        while not h.done:
            beams.append(h.beams)
            st.step()
            reqs, logits = st.last_logits
            rows.append(logits[[i for i, r in enumerate(reqs) if r.id == h.id]].clone())
        return rows, beams, list(h.tokens), h.score, list(h.slots)
    finally:
        st.close()


@pytest.mark.parametrize("kind", ["bf16", "fp16", "nf4"])
@pytest.mark.parametrize("mode", ["sample", "beam2", "beam4"])
def test_request_does_not_depend_on_admission_slot_or_neighbours(model, ops, kind, mode):
    V, cfg, sd = model
    eng = engine(model, kind)
    reqs = requests(cfg, eng.dtype, 4)
    target = reqs[0]
    tkw = SAMPLED if mode == "sample" else dict(num_beams=int(mode[-1]))
    other_k = 4 if mode == "beam2" else 2
    fillers = [(reqs[1], 3, {}), (reqs[2], 70, dict(SAMPLED, seed=9)), (reqs[3], 70, dict(num_beams=other_k))]
    with ops.batch_invariant():
        alone = run_target(eng, target, tkw, [], 0, 6)
        slots = {tuple(alone[4])}
        for s in (0, 1, 7):
            got = run_target(eng, target, tkw, fillers, s, 6)
            slots.add(tuple(got[4]))
            assert len(got[0]) == len(alone[0])
            for a, b in zip(got[0], alone[0]):
                assert torch.equal(a, b), (kind, mode, s)
            assert got[1:4] == alone[1:4], (kind, mode, s)
    assert len(slots) >= 2                       # other slots, and a retired filler's slot reused (s = 7)


@pytest.mark.parametrize("kind", ["bf16", "fp16", "nf4"])
def test_sampled_tokens_follow_the_oracle_on_stream_logits(model, ops, kind):
    V, cfg, sd = model
    eng = engine(model, kind)
    reqs = requests(cfg, eng.dtype, 3, seed=21)
    loose = total = 0
    for i, (T, k, p) in enumerate(((0.7, 50, 0.9), (1.0, 0, None), (1.5, 5, 0.5))):
        fillers = [(reqs[(i + 1) % 3], 9, {}), (reqs[(i + 2) % 3], 9, dict(num_beams=2))]
        seed = 1000 + i
        rows, _, toks, _, _ = run_target(eng, reqs[i], dict(temperature=T, top_k=k, top_p=p, seed=seed), fillers, 1, 8)
        assert len(toks) == 9
        for step, (row, t) in enumerate(zip(rows, toks)):
            r = S.sample_row(row[0].cpu(), T, k, p, eng.dtype, seed, step)
            if r["token"] != t:
                assert r["margin"] < MARGIN, (i, step, t, r["token"], r["margin"])
                loose += 1
            total += 1
    assert loose <= 1, (loose, total)


@pytest.mark.parametrize("kind", ["bf16", "fp16", "nf4"])
@pytest.mark.parametrize("k,eos,kw", [(2, -1, {}), (3, 7, dict(length_penalty=0.5)), (4, 11, dict(early_stopping=True)),
                                      (4, 13, dict(early_stopping="never", length_penalty=2.0))])
def test_beam_request_matches_the_oracle_on_stream_logits(model, ops, kind, k, eos, kw):
    V, cfg, sd = model
    eng = engine(model, kind)
    reqs = requests(cfg, eng.dtype, 3, seed=30 + k)
    N = 7
    for s in range(2):
        target = reqs[s]
        fillers = [(reqs[2], 12, dict(SAMPLED, seed=5)), (reqs[1 - s], 12, dict(num_beams=2))]
        rows, beams, ids, score, _ = run_target(eng, target, dict(num_beams=k, **kw), fillers, s, N - 1, slots=k + 4, eos=eos)

        def step_logits(step, bs):
            assert bs == beams[step], (step, bs, beams[step])
            return rows[step].float().cpu()

        res = BO.beam_search(step_logits, len(target[0]), k, N, eos, eng.dtype, **kw)
        if (ids, score) != (res["ids"], res["score"]):
            assert BO.min_margin(res) < MARGIN, (s, ids, res["ids"], score, res["score"])


def test_top_k_1_is_greedy_on_the_stream(model, ops):
    V, cfg, sd = model
    eng = engine(model, "bf16")
    reqs = requests(cfg, BF, 3, seed=2)
    with ops.batch_invariant():                  # the neighbour changes the batch, so the logits are compared batch-invariant
        for r in reqs:
            rows, _, greedy, _, _ = run_target(eng, r, {}, [], 0, 7)
            for T in (0.3, 1.0, 2.0):
                sampled = run_target(eng, r, dict(temperature=T, top_k=1, seed=77), [(reqs[0], 4, {})], 1, 7)[2]
                if sampled != greedy:
                    # only where the fp32 argmax and a token tied with it after rounding to the engine dtype part ways
                    j = next(i for i in range(len(greedy)) if sampled[i] != greedy[i])
                    v = S.scale(rows[j][0].cpu(), T, BF)
                    assert v[sampled[j]] == v[greedy[j]] == v.max(), (T, j)


# ------------------------------------------------------------------------------------------------ end to end
def items(n=5):
    from PIL import Image
    rng = np.random.default_rng(4)
    out = []
    for i in range(n):
        img = Image.fromarray(rng.integers(0, 256, (60 + 10 * i, 80, 3), dtype=np.uint8), "RGB")
        out.append((img, " ".join(["word"] * (1 + i)), None, None, None))
    return out


@pytest.mark.parametrize("kind", ["bf16", "nf4"])
def test_sampled_stream_equals_free_form_inference(model, ops, kind):
    from vstar_b200.vqa import VQA_LLM
    llm = VQA_LLM(engine=engine(model, kind))
    its = items()
    with ops.batch_invariant():
        for T, p in ((0.7, 0.9), (1.3, None)):
            torch.manual_seed(11)
            got = dict(llm.free_form_inference_stream(its, max_new_tokens=6, slots=2, temperature=T, top_p=p))
            torch.manual_seed(11)
            want = {i: llm.free_form_inference(it[0], it[1], temperature=T, top_p=p, max_new_tokens=6) for i, it in enumerate(its)}
            assert got == want, (T, p)


def test_beam_stream_equals_free_form_inference(model, ops):
    from vstar_b200.vqa import VQA_LLM
    llm = VQA_LLM(engine=engine(model, "bf16"))
    its = items(4)
    with ops.batch_invariant():
        got = dict(llm.free_form_inference_stream(its, max_new_tokens=5, slots=5, num_beams=2))
        want = {i: llm.free_form_inference(it[0], it[1], num_beams=2, max_new_tokens=5) for i, it in enumerate(its)}
    assert got == want
    with pytest.raises(ValueError):
        list(llm.free_form_inference_stream(its, max_new_tokens=5, slots=2, num_beams=3))


def parent_step(st):
    """the greedy step of the parent commit, for the launch-sequence comparison"""
    from vstar_b200 import ops
    act = st.active
    e, c = st.engine, st.engine.cfg
    lens = [r.prompt_len + len(r.tokens) - 1 for r in act]
    meta = torch.tensor([[r.slot for r in act], lens, lens], dtype=torch.int32).to(e.dev)
    ids = torch.tensor([r.tokens[-1] for r in act], dtype=torch.int64).to(e.dev)
    x = ops.gather_rows(ids, e.w.embed)
    ops.llama_layers_slots(e._layer_table, len(e.w.layers), x, st._cache, c.rms_eps, e.w.rope_cos, e.w.rope_sin, st._scratch,
                           meta[0], meta[1], meta[2], max(lens), c.n_heads, c.intermediate,
                           norm_folded=getattr(e.w, "fold_norms", False), deq_scratch=st._deq)
    hn = ops.rmsnorm(x, e.w.final_norm, c.rms_eps)
    logits = ops.gemm(hn, e.w.lm_head, out_dtype=torch.float32)
    nxt = ops.argmax_rows(logits)[0].tolist()
    for r, t in zip(act, nxt):
        r.tokens.append(int(t))
        if st._ended(r):
            r.done = True
            st._slots[r.slot] = None
    return logits


@pytest.mark.parametrize("kind", ["bf16", "nf4"])
def test_greedy_stream_issues_the_parent_launches(model, ops, monkeypatch, kind):
    from vstar_b200 import _lib
    V, cfg, sd = model
    eng = engine(model, kind)
    reqs = requests(cfg, eng.dtype, 4, seed=13)
    calls = []
    real = ops.call
    monkeypatch.setattr(ops, "call", lambda name, *a: (calls.append(name), real(name, *a))[1])

    def run(step):
        st = eng.decode_stream(3, max_positions=400, eos_token_id=-1)
        per, logits, pending = [], [], list(zip(reqs, (3, 6, 4, 5)))
        while pending and st.free_slots:
            st.admit(*pending.pop(0))
        while st.active:
            n0, calls[:] = _lib.launches, []
            lg = step(st)
            per.append((_lib.launches - n0, list(calls)))
            logits.append(lg.clone())
            while pending and st.free_slots:
                st.admit(*pending.pop(0))
        st.close()
        return per, logits

    def now(st):
        st.step()
        return st.last_logits[1]

    want = run(parent_step)
    got = run(now)
    assert got[0] == want[0]
    assert len(got[1]) == len(want[1]) and all(torch.equal(a, b) for a, b in zip(got[1], want[1]))


def test_mixed_step_makes_one_device_to_host_copy(model, ops):
    from torch.profiler import ProfilerActivity, profile
    V, cfg, sd = model
    eng = engine(model, "bf16")
    reqs = requests(cfg, BF, 4, seed=17)
    st = eng.decode_stream(9, max_positions=400, eos_token_id=-1)
    st.admit(reqs[0], 8)
    st.admit(reqs[1], 8, **SAMPLED)
    st.admit(reqs[2], 8, num_beams=2)
    st.admit(reqs[3], 8, num_beams=4)
    st.step()
    st.step()                                   # forks copy rows from here on
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        st.step()
        torch.cuda.synchronize()
    st.close()
    d2h = sum(e.count for e in prof.key_averages() if "DtoH" in e.key)
    assert d2h == 1, [(e.key, e.count) for e in prof.key_averages() if "Memcpy" in e.key]


def test_mixed_stream_close_returns_device_memory(model, ops):
    V, cfg, sd = model
    eng = engine(model, "fp16")
    reqs = requests(cfg, F16, 3)
    eng.decode_stream(1, max_positions=64).close()
    gc.collect()
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    st = eng.decode_stream(7, max_positions=512, eos_token_id=-1)
    st.admit(reqs[0], 4, **SAMPLED)
    st.admit(reqs[1], 5, num_beams=4)
    st.admit(reqs[2], 3)
    while st.active:
        st.step()
    st.close()
    del st
    gc.collect()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == m0


def test_admission_refusals_raise_before_any_launch(model, ops):
    from vstar_b200 import _lib
    V, cfg, sd = model
    eng = engine(model, "bf16")
    reqs = requests(cfg, BF, 2)
    st = eng.decode_stream(3, max_positions=300, eos_token_id=2)
    st.admit(reqs[0], 4)
    n0 = _lib.launches
    for kw, exc in ((dict(num_beams=2, temperature=0.7), NotImplementedError), (dict(num_beams=2, stop_ids=[5]), ValueError),
                    (dict(num_beams=17), ValueError), (dict(num_beams=4), ValueError), (dict(num_beams=3), RuntimeError),
                    (dict(temperature=0.7, top_p=1.5), ValueError), (dict(temperature=0.7, top_k=-1), ValueError)):
        with pytest.raises(exc):
            st.admit(reqs[1], 4, **kw)
    T = eng.spliced_length(reqs[1][0], 0, reqs[1][3])
    with pytest.raises(_lib.VsbError, match="exceeds"):
        st.admit(reqs[1], 300 - T + 1, num_beams=2)
    assert _lib.launches == n0
    h = st.admit(reqs[1], 4, num_beams=2, stop_ids=[2])
    assert len(h.slots) == 2 and st.free_slots == 0
    st.close()
