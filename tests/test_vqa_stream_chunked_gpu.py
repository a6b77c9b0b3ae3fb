"""Chunked prefill on the paged decode stream (DecodeStream(kv_pages=N, prefill_chunk=C)).

(1) vsb_attn_chunk_paged == rows [lo, lo + n) of one causal vsb_flash_attn over the same contiguous keys [0, lo + n), bit for
    bit (pages in random order, every other page row NaN, several segments per launch, a pool of two layers); float64 where
    lo + n < 64 (vsb_flash_attn then runs its mma.sync kernel);
(2) vsb_llama_layers_chunked_paged: decode rows == vsb_llama_layers_slots_paged, chunk rows' final hidden states == the one-shot
    vsb_llama_layers prefill, bf16 (folded), f16 and NF4, batch-invariant mode;
(3) greedy, sampled and beam requests give the unchunked paged stream's tokens, beam scores, first-token and per-step logits for
    every C, and running requests gain one token per step while prompts prefill, at most C prompt rows per step;
(4) the stream's device memory is its pool, page table, scratch and held embeddings; free_form_inference_stream(prefill_chunk=)
    equals the call without it."""
import gc

import numpy as np
import pytest
import torch

from tests.test_vqa_stream_gpu import bits, engine, model, ops, randn, requests  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu
BF, F16 = torch.bfloat16, torch.float16


def attn_ref64(q, k, v, H, D, lo):
    """float64 causal attention of query rows lo.. over keys [0, lo + i]"""
    n, T = q.shape[0], k.shape[0]
    qd, kd, vd = (t.double().cpu().view(-1, H, D) for t in (q, k, v))
    s = torch.einsum("qhd,khd->hqk", qd, kd) * D ** -0.5
    mask = torch.arange(T)[None, :] > (lo + torch.arange(n))[:, None]
    p = torch.softmax(s.masked_fill(mask, float("-inf")), -1)
    return torch.einsum("hqk,khd->qhd", p, vd).reshape(n, H * D)


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("dt", [BF, F16])
@pytest.mark.parametrize("H,D", [(2, 128), (3, 64)])
@pytest.mark.parametrize("n", [1, 17, 64, 200])
def test_chunk_attention_equals_flash_attention(ops, dt, H, D, n):
    los = [0, 1, 63, 64, 65, 127, 128, 300]
    P, HD, S = 64, H * D, len(los)
    ppr = -(-(max(los) + n) // P)
    n_pages = S * ppr + 5
    g = torch.Generator().manual_seed(n + D)
    perm = torch.randperm(n_pages, generator=g).tolist()
    pool = torch.full((2, n_pages, P, 2 * HD), float("nan"), dtype=dt)            # layer 0 stays NaN; the keys live in layer 1
    table = torch.zeros((S + 2, ppr), dtype=torch.int32)
    slots = torch.randperm(S + 2, generator=g)[:S].tolist()
    ldq = HD + 64
    q = torch.full((n * S, ldq), float("nan"), dtype=dt)
    seqs, k = [], 0
    for s, lo in enumerate(los):
        T = lo + n
        seq = (randn(T, 3 * HD, seed=100 * s + n) * 2).to(dt)
        seqs.append(seq)
        for j in range(-(-T // P)):
            table[slots[s], j] = perm[k]
            rows = seq[j * P:min((j + 1) * P, T), HD:]
            pool[1, perm[k], :rows.shape[0]] = rows
            k += 1
        q[s * n:(s + 1) * n, :HD] = seq[lo:, :HD]
    seg = torch.tensor([slots, los, [n] * S], dtype=torch.int32).cuda()
    pool, table, q = pool.cuda(), table.cuda(), q.cuda()
    out = torch.empty((n * S, HD), dtype=dt, device="cuda")
    ops.attn_chunk_paged(q[:, :HD], pool, table, out, H, D, D ** -0.5, seg, layer=1)
    torch.cuda.synchronize()
    assert not torch.isnan(out).any()
    ulp = 2.0 ** -8 if dt == BF else 2.0 ** -11
    for s, lo in enumerate(los):
        T = lo + n
        got = out[s * n:(s + 1) * n]
        if T >= 64:
            seq = seqs[s].cuda()
            want = torch.empty((T, HD), dtype=dt, device="cuda")
            ops.flash_attn(seq, seq[:, HD:], seq[:, 2 * HD:], want, 1, H, T, T, D, True, D ** -0.5, T * 3 * HD, 3 * HD, T * 3 * HD,
                           3 * HD, T * 3 * HD, 3 * HD, T * HD, HD)
            torch.cuda.synchronize()
            assert torch.equal(bits(got), bits(want[lo:])), (lo, n)
        else:
            seq = seqs[s]
            ref = attn_ref64(seq[lo:, :HD], seq[:, HD:2 * HD], seq[:, 2 * HD:], H, D, lo)
            err = (got.double().cpu() - ref).abs()
            assert bool((err <= 2 * ulp * ref.abs() + 4 * ulp * ref.abs().max()).all()), (lo, n, float(err.max()))


def test_chunk_attention_refuses_pages_of_other_than_64k_rows(ops):
    from vstar_b200 import _lib
    pool = torch.zeros((4, 32, 2 * 128), dtype=BF, device="cuda")
    table = torch.zeros((2, 4), dtype=torch.int32, device="cuda")
    seg = torch.tensor([[0], [0], [8]], dtype=torch.int32, device="cuda")
    q = torch.zeros((8, 128), dtype=BF, device="cuda")
    out = torch.empty_like(q)
    with pytest.raises(_lib.VsbError, match="multiple of 64"):
        ops.attn_chunk_paged(q, pool, table, out, 1, 128, 0.1, seg)


# ------------------------------------------------------------------------------------------------ runner
def paged_pool(cache, P, n_pages, gen):
    """cache [L, Bc, Tmax, 3d] -> (pool [L, n_pages, P, 2d] of its k|v rows in randomly ordered pages, NaN elsewhere; table)"""
    L, Bc, Tmax, W = cache.shape
    d = W // 3
    ppr = Tmax // P
    perm = torch.randperm(n_pages, generator=gen)
    table = torch.zeros((Bc, ppr), dtype=torch.int32)
    pool = torch.full((L, n_pages, P, 2 * d), float("nan"), dtype=cache.dtype, device=cache.device)
    for s in range(Bc):
        for j in range(ppr):
            p = int(perm[s * ppr + j])
            table[s, j] = p
            pool[:, p] = cache[:, s, j * P:(j + 1) * P, d:]
    return pool, table.cuda()


@pytest.mark.parametrize("kind", ["bf16", "fp16", "nf4"])
def test_chunked_runner_equals_slot_runner_and_prefill(model, ops, kind):
    V, cfg, sd = model
    eng = engine(model, kind)
    if eng._layer_table is None:
        eng._layer_table = ops.llama_layer_table(eng.w.layers)
    c, dt = eng.cfg, eng.dtype
    L, d, P, inter = c.n_layers, c.hidden, 64, c.intermediate
    folded = getattr(eng.w, "fold_norms", False)
    deq = torch.empty((2 * inter * d,), dtype=dt, device="cuda") if kind == "nf4" else None
    lengths = [63, 64, 300]                                  # decode rows on page-table rows 0..2; prompts on rows 3 and 4
    Bc, Tmax = 5, 768
    cache = (randn(L, Bc, Tmax, 3 * d, seed=2) * 0.5).to(dt).cuda()
    pool, table = paged_pool(cache, P, Bc * Tmax // P + 3, torch.Generator().manual_seed(6))
    prompts = [(3, (randn(300, d, seed=7) * 0.5).to(dt).cuda()), (4, (randn(70, d, seed=8) * 0.5).to(dt).cuda())]
    with ops.batch_invariant():
        want = []                                            # one-shot prefill of each prompt
        for _, xp in prompts:
            T = xp.shape[0]
            x = xp.clone()
            stage = torch.empty((L, 1, T, 3 * d), dtype=dt, device="cuda")
            ops.llama_layers(eng._layer_table, L, x, 1, T, 0, stage, 1, T, d, c.n_heads, inter, c.rms_eps, eng.w.rope_cos, eng.w.rope_sin,
                             torch.empty((T * (2 * d + inter),), dtype=dt, device="cuda"), norm_folded=folded, deq_scratch=deq)
            want.append(x)
        got = [torch.empty_like(xp) for _, xp in prompts]
        # step 1: rows [0, 150) of prompt 0; step 2: rows [150, 300) of prompt 0 and all 70 rows of prompt 1
        plan = [[(0, 0, 150)], [(0, 150, 150), (1, 0, 70)]]
        for step, segs in enumerate(plan):
            lens = [n + step for n in lengths]
            B, R = len(lens), sum(n for _, _, n in segs)
            x0 = randn(B, d, seed=10 + step).to(dt).cuda()
            ref_pool = pool.clone()
            xr = x0.clone()
            sl = torch.tensor([0, 1, 2], dtype=torch.int32, device="cuda")
            ln = torch.tensor(lens, dtype=torch.int32, device="cuda")
            ops.llama_layers_slots_paged(eng._layer_table, L, xr, ref_pool, table, c.rms_eps, eng.w.rope_cos, eng.w.rope_sin,
                                         torch.empty((B * (5 * d + inter),), dtype=dt, device="cuda"), sl, ln, ln, max(lens), c.n_heads,
                                         inter, norm_folded=folded, deq_scratch=deq)
            x = torch.cat([x0] + [prompts[i][1][lo:lo + n] for i, lo, n in segs]).contiguous()
            slot = torch.tensor([0, 1, 2] + [prompts[i][0] for i, lo, n in segs for _ in range(n)], dtype=torch.int32, device="cuda")
            ln = torch.tensor(lens + [lo + j for i, lo, n in segs for j in range(n)], dtype=torch.int32, device="cuda")
            seg = torch.tensor([[prompts[i][0] for i, _, _ in segs], [lo for _, lo, _ in segs], [n for _, _, n in segs]],
                               dtype=torch.int32, device="cuda")
            ops.llama_layers_chunked_paged(eng._layer_table, L, x, pool, table, c.rms_eps, eng.w.rope_cos, eng.w.rope_sin,
                                           torch.empty(((B + R) * (5 * d + inter),), dtype=dt, device="cuda"), slot, ln, ln, max(lens), seg,
                                           R, c.n_heads, inter, norm_folded=folded, deq_scratch=deq)
            torch.cuda.synchronize()
            assert torch.equal(bits(x[:B]), bits(xr))                                # decode rows: the slot runner's bits
            o = B
            for i, lo, n in segs:
                got[i][lo:lo + n] = x[o:o + n]
                o += n
    for g, w in zip(got, want):
        assert torch.equal(bits(g), bits(w))                                        # chunk rows: the one-shot prefill's bits


# ------------------------------------------------------------------------------------------------ streams
def long_requests(cfg, dt, n, seed):
    """requests whose prompts are >= 64 rows (the long image: 256 rows)"""
    return [(ids, img, crops, [True], ol) for ids, img, crops, _, ol in requests(cfg, dt, n, seed=seed)]


SETTINGS = [dict(), dict(temperature=0.8, top_k=20, top_p=0.9, seed=11), dict(num_beams=2), dict(), dict(num_beams=4),
            dict(temperature=1.1, seed=-5), dict(num_beams=2), dict()]


def run_stream(st, reqs, budgets, settings, C=None):
    """admit requests in order whenever their slots and pages are free -> ({request: tokens}, {request: beam score},
    {request: [logits rows of that request, per call]}, steps where running requests and prompt rows shared the step)"""
    out, score, logits, owner, nxt, shared = {}, {}, {}, {}, 0, 0
    lens = [st.engine.spliced_length(r[0], 0, r[3]) for r in reqs]

    def record():
        if st.last_logits is None:
            return
        rs, lg = st.last_logits
        for i, r in enumerate(rs):
            logits.setdefault(owner[r.id], []).append(lg[i].clone())

    def admit_all():
        nonlocal nxt
        while nxt < len(reqs):
            k = settings[nxt].get("num_beams", 1)
            if st.free_slots < k or st.pages.need(lens[nxt], budgets[nxt], k) > st.pages.free_pages:
                break
            h = st.admit(reqs[nxt], budgets[nxt], **settings[nxt])
            owner[h.id] = nxt
            nxt += 1
            if C is None:
                record()
    admit_all()
    while len(out) < len(reqs):
        running = [r for r in st.active if not r.prefilling]
        before = {r.id: len(r.tokens) if r.beam is None else len(r.beam.beams[0]) for r in running}
        filled = {r.id: r.prefilled for r in st.active}
        ended = st.step()
        for r, toks in ended:
            out[owner[r.id]] = list(toks)
            score[owner[r.id]] = r.score
        record()
        if C is not None:
            rows = sum(r.prefilled - filled[r.id] for r in st.active + [r for r, _ in ended] if r.id in filled)
            assert rows <= C
            shared += bool(rows and running)
            for r in running:                                # a running request gains one token every step, whatever prefills
                if not r.done:
                    assert (len(r.tokens) if r.beam is None else len(r.beam.beams[0])) == before[r.id] + 1
        admit_all()
    return out, score, logits, shared


@pytest.mark.parametrize("kind", ["bf16", "fp16", "nf4"])
def test_chunked_stream_equals_unchunked_stream(model, ops, kind):
    V, cfg, sd = model
    eng = engine(model, kind)
    reqs = long_requests(cfg, eng.dtype, 8, seed=21)
    budgets = [9, 5, 7, 12, 6, 10, 4, 8]
    longest = max(eng.spliced_length(r[0], 0, r[3]) for r in reqs)
    with ops.batch_invariant():
        st = eng.decode_stream(6, max_positions=512, eos_token_id=-1, kv_pages=6 * 8)
        try:
            want = run_stream(st, reqs, budgets, SETTINGS)
        finally:
            st.close()
        for C in (64, 100, 256, longest + 1):
            st = eng.decode_stream(6, max_positions=512, eos_token_id=-1, kv_pages=6 * 8, prefill_chunk=C)
            try:
                got = run_stream(st, reqs, budgets, SETTINGS, C=C)
                assert st.pages.free_pages == st.pages.n_pages and not st._prefilling
            finally:
                st.close()
            assert got[0] == want[0], C
            assert got[1] == want[1], C
            assert sorted(got[2]) == sorted(want[2])
            for i in want[2]:
                assert len(got[2][i]) == len(want[2][i]), (C, i)
                for a, b in zip(got[2][i], want[2][i]):
                    assert torch.equal(a, b), (C, i)
            if C < longest:
                assert got[3] > 0                            # some step carried running rows and prompt rows together


def _requested():
    return torch.cuda.memory_stats()["requested_bytes.all.current"]


def test_chunked_stream_device_memory_is_pool_table_scratch_and_embeddings(model, ops):
    V, cfg, sd = model
    eng = engine(model, "bf16")
    reqs = long_requests(cfg, BF, 2, seed=3)
    with eng.decode_stream(1, max_positions=512, kv_pages=8, prefill_chunk=64) as st:  # warms the layer table and CLIP
        st.admit(reqs[0], 2)
        while st.active:
            st.step()
    gc.collect()
    torch.cuda.synchronize()
    m0, r0 = torch.cuda.memory_allocated(), _requested()
    slots, Tm, N, C, c = 3, 512, 20, 100, cfg
    st = eng.decode_stream(slots, max_positions=Tm, eos_token_id=-1, kv_pages=N, prefill_chunk=C)
    pool = c.n_layers * N * 64 * 2 * c.hidden * 2
    scratch = (slots + C) * (5 * c.hidden + c.intermediate) * 2
    table = slots * (Tm // 64) * 4
    assert _requested() - r0 == pool + scratch + table
    held = 0
    for r in reqs:
        h = st.admit(r, 4)
        held += h.prompt_len * c.hidden * 2
        assert h.prefilling and h.tokens == [] and h.prefilled == 0
        gc.collect()
        assert _requested() - r0 == pool + scratch + table + held       # no staging cache: the embeddings wait on the device
    while st.active:
        st.step()
    assert st.pages.free_pages == N and all(getattr(h, "_x", None) is None for h in st._prefilling) and not st._prefilling
    st.close()
    del st
    gc.collect()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == m0


def test_chunked_free_form_inference_stream_equals_unchunked(model, ops):
    from PIL import Image
    from vstar_b200.vqa import VQA_LLM
    V, cfg, sd = model
    llm = VQA_LLM(engine=engine(model, "bf16"))
    rng = np.random.default_rng(4)
    items = []
    for i in range(5):
        img = Image.fromarray(rng.integers(0, 256, (60 + 10 * i, 80, 3), dtype=np.uint8), "RGB")
        items.append((img, " ".join(["word"] * (1 + i)), None, None, None))
    with ops.batch_invariant():
        want = dict(llm.free_form_inference_stream(items, max_new_tokens=6, slots=4, kv_pages=24))
        got = dict(llm.free_form_inference_stream(items, max_new_tokens=6, slots=4, kv_pages=24, prefill_chunk=128))
        beams = dict(llm.free_form_inference_stream(items, max_new_tokens=6, slots=4, num_beams=2, kv_pages=24))
        beams_c = dict(llm.free_form_inference_stream(items, max_new_tokens=6, slots=4, num_beams=2, kv_pages=24, prefill_chunk=100))
    assert got == want and beams_c == beams
