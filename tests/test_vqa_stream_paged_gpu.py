"""Paged decode stream (DecodeStream(kv_pages=N)): the KV cache as a pool of k|v pages found through a page table.

(1) vsb_rope_scatter_paged and vsb_attn_decode_paged == vsb_rope_scatter and vsb_attn_decode_slots bit for bit on the same
    logical cache (pages in random order, page-boundary lengths, every split count, both modes);
(2) vsb_llama_layers_slots_paged == vsb_llama_layers_slots bit for bit for bf16 (folded norms), f16 and NF4 layer tables;
(3) the same admission schedule of greedy, sampled and beam (k = 2, 4) requests on a contiguous and a paged stream gives the same
    tokens and bit-identical logits at every admission and step, in bf16, fp16 and NF4;
(4) a pool of the bytes of S contiguous slots holds more than S requests at once, with the contiguous stream's answers in
    batch-invariant mode; the stream's device memory is its pool, scratch and page table; free_form_inference_stream(kv_pages=)
    equals the contiguous call."""
import gc

import numpy as np
import pytest
import torch

from tests.test_vqa_stream_gpu import bits, engine, model, ops, randn, requests, rope_tables  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu
BF, F16 = torch.bfloat16, torch.float16


def paged_copy(cache, lengths_cap, P, n_pages, gen):
    """the k|v rows [0, cap) of every slot of cache [Bc, Tmax, 3HD] in a pool [n_pages, P, 2HD] of randomly ordered pages ->
    (pool, page table int32 [Bc, ceil(Tmax / P)] on the device).  Unused pages hold NaN."""
    Bc, Tmax, W = cache.shape
    HD = W // 3
    ppr = -(-Tmax // P)
    perm = torch.randperm(n_pages, generator=gen)
    table = torch.zeros((Bc, ppr), dtype=torch.int32)
    pool = torch.full((n_pages, P, 2 * HD), float("nan"), dtype=cache.dtype, device=cache.device)
    k = 0
    for s in range(Bc):
        for j in range(-(-lengths_cap // P)):
            table[s, j] = int(perm[k])
            rows = cache[s, j * P:min((j + 1) * P, Tmax), HD:]
            pool[int(perm[k]), :rows.shape[0]] = rows
            k += 1
    return pool, table.cuda()


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("invariant", [False, True])
@pytest.mark.parametrize("P", [16, 64])
@pytest.mark.parametrize("dt", [BF, F16])
@pytest.mark.parametrize("H,D", [(2, 128), (3, 64)])
def test_paged_rope_scatter_and_attention_equal_the_slot_kernels(ops, H, D, dt, P, invariant):
    lengths = [0, P - 1, P, P + 1, 127, 255, 511, 1500]           # 1..8 splits by the key-count rule
    B, Bc, Tmax = len(lengths), len(lengths) + 3, 1536
    HD, W = H * D, 3 * H * D
    g = torch.Generator().manual_seed(H * D + P)
    slot = torch.randperm(Bc, generator=g)[:B].to(torch.int32).cuda()
    length = torch.tensor(lengths, dtype=torch.int32).cuda()
    pos = torch.tensor([n + 3 for n in lengths], dtype=torch.int32).cuda()
    cos, sin = rope_tables(2048, D, dt)
    cache = randn(Bc, Tmax, W, seed=P + D).to(dt).cuda()
    pool, table = paged_copy(cache, Tmax, P, Bc * (-(-Tmax // P)) + 5, g)
    qkv = randn(B, W + 8, seed=7).to(dt).cuda()[:, :W]
    q_paged = qkv.clone()
    ops.rope_scatter(qkv.contiguous(), cache, H, D, cos, sin, slot, length, pos)
    ops.rope_scatter_paged(q_paged, pool, table, H, D, cos, sin, slot, length, pos)
    torch.cuda.synchronize()
    for b, (s, n) in enumerate(zip(slot.tolist(), lengths)):
        row = cache[s, n]
        assert torch.equal(bits(q_paged[b, :HD]), bits(row[:HD]))                  # q rotated in place
        assert torch.equal(bits(q_paged[b, HD:]), bits(qkv[b, HD:]))               # k|v of the scratch row untouched
        page = int(table[s, n // P])
        assert torch.equal(bits(pool[page, n % P]), bits(row[HD:]))               # rotated k and v in the row's page
    want = torch.empty((B, HD), dtype=dt, device="cuda")
    got = torch.empty((B, HD), dtype=dt, device="cuda")
    ctx = ops.batch_invariant() if invariant else torch.no_grad()
    with ctx:
        ops.attn_decode_slots(cache, want, H, D, D ** -0.5, slot, length, max_len=1500)
        ops.attn_decode_paged(q_paged, pool, table, got, H, D, D ** -0.5, slot, length, max_len=1500)
        torch.cuda.synchronize()
        assert torch.equal(bits(got), bits(want))
        if invariant:                                                               # each row alone, too
            for b in (0, B - 1):
                one = torch.empty((1, HD), dtype=dt, device="cuda")
                ops.attn_decode_paged(q_paged[b:b + 1], pool, table, one, H, D, D ** -0.5, slot[b:b + 1], length[b:b + 1])
                assert torch.equal(bits(one[0]), bits(want[b]))


def test_paged_copy_equals_slot_copy(ops):
    """a beam fork's ranged copy between page-table rows == vsb_copy_slot_rows_b16 on the same logical rows; a contiguous
    source writes a prompt into pages; the slot rules refuse before any launch"""
    from vstar_b200 import _lib
    L, Bc, Tmax, HD, P = 3, 6, 300, 64, 16
    g = torch.Generator().manual_seed(3)
    cache = randn(L, Bc, Tmax, 3 * HD, seed=4).to(BF).cuda()
    pools, table = [], None
    for li in range(L):
        gl = torch.Generator().manual_seed(9)                                       # the same page order in every layer
        p, table = paged_copy(cache[li], Tmax, P, Bc * (-(-Tmax // P)), gl)
        pools.append(p)
    pool = torch.stack(pools)
    quads = [(0, 2, 5, 70), (1, 3, 0, 300), (4, 5, 17, 18)]
    ops.copy_slot_rows(cache, quads)
    ops.copy_page_rows(pool, table, quads)
    src = randn(L, 2, 100, 3 * HD, seed=5).to(BF).cuda()
    ops.copy_page_rows(pool, table, [(1, 0, 0, 100), (0, 1, 33, 100)], src=src[..., HD:])
    cache[:, 0, :100] = src[:, 1]
    cache[:, 1, 33:100] = src[:, 0, 33:]
    torch.cuda.synchronize()
    tab = table.cpu()
    for s in range(Bc):
        for n in range(Tmax):
            if n % 37 and n not in (5, 69, 70, 17, 99, 100):
                continue
            page = int(tab[s, n // P])
            assert torch.equal(bits(pool[:, page, n % P]), bits(cache[:, s, n, HD:])), (s, n)
    n0 = _lib.launches
    for bad in ([(0, 1, 0, 5), (1, 2, 0, 5)], [(0, 2, 0, 5), (1, 2, 0, 5)], [(0, Bc, 0, 5)], [(0, 1, 5, 4)],
                [(0, 1, 0, 1 + (-(-Tmax // P)) * P)]):
        with pytest.raises(_lib.VsbError):
            ops.copy_page_rows(pool, table, bad)
    assert _lib.launches == n0 + 5                                                  # counted, refused by the library before launch


@pytest.mark.parametrize("kind", ["bf16", "fp16", "nf4"])
def test_paged_runner_equals_slot_runner(model, ops, kind):
    V, cfg, sd = model
    eng = engine(model, kind)
    if eng._layer_table is None:
        eng._layer_table = ops.llama_layer_table(eng.w.layers)
    c, dt = eng.cfg, eng.dtype
    L, d, P = c.n_layers, c.hidden, 64
    lengths = [0, 63, 64, 65, 300, 700]
    B, Bc, Tmax = len(lengths), len(lengths) + 2, 768
    g = torch.Generator().manual_seed(1)
    cache = (randn(L, Bc, Tmax, 3 * d, seed=2) * 0.5).to(dt).cuda()
    pools, table = [], None
    for li in range(L):
        pl, table = paged_copy(cache[li], Tmax, P, Bc * (Tmax // P) + 3, torch.Generator().manual_seed(6))
        pools.append(pl)
    pool = torch.stack(pools)
    slot = torch.randperm(Bc, generator=g)[:B].to(torch.int32).cuda()
    length = torch.tensor(lengths, dtype=torch.int32).cuda()
    x0 = (randn(B, d, seed=3)).to(dt).cuda()
    deq = torch.empty((2 * c.intermediate * d,), dtype=dt, device="cuda") if kind == "nf4" else None
    folded = getattr(eng.w, "fold_norms", False)
    if kind == "bf16":
        assert folded
    outs = []
    for paged in (False, True):
        x = x0.clone()
        scratch = torch.empty((B * (5 * d + c.intermediate),), dtype=dt, device="cuda")
        if paged:
            ops.llama_layers_slots_paged(eng._layer_table, L, x, pool, table, c.rms_eps, eng.w.rope_cos, eng.w.rope_sin, scratch, slot,
                                         length, length, max(lengths), c.n_heads, c.intermediate, norm_folded=folded, deq_scratch=deq)
        else:
            ops.llama_layers_slots(eng._layer_table, L, x, cache, c.rms_eps, eng.w.rope_cos, eng.w.rope_sin, scratch, slot, length,
                                   length, max(lengths), c.n_heads, c.intermediate, norm_folded=folded, deq_scratch=deq)
        outs.append(x)
    torch.cuda.synchronize()
    assert torch.equal(bits(outs[0]), bits(outs[1]))
    tab = table.cpu()
    for s, n in zip(slot.tolist(), lengths):                                        # the new k|v rows of every layer
        assert torch.equal(bits(pool[:, int(tab[s, n // P]), n % P]), bits(cache[:, s, n, d:]))


# ------------------------------------------------------------------------------------------------ streams
def mixed_settings(n):
    kinds = [dict(), dict(temperature=0.8, top_k=20, top_p=0.9, seed=11), dict(num_beams=2), dict(),
             dict(num_beams=4), dict(temperature=1.1, seed=-5), dict(num_beams=2), dict()]
    return [kinds[i % len(kinds)] for i in range(n)]


def drive(st, reqs, budgets, settings, fits=None):
    """admit requests in order whenever their slots (and pages) are free; -> (trace of (request ids, logits) after every
    admission and step, {request index: tokens}, most requests running at once)"""
    trace, out, owner, nxt, most = [], {}, {}, 0, 0

    def can():
        k = settings[nxt].get("num_beams", 1)
        return st.free_slots >= k and (fits is None or fits(nxt))

    def admit_all():
        nonlocal nxt
        while nxt < len(reqs) and can():
            h = st.admit(reqs[nxt], budgets[nxt], **settings[nxt])
            owner[h.id] = nxt
            rs, lg = st.last_logits
            trace.append(([r.id for r in rs], lg.clone()))
            nxt += 1
    admit_all()
    while len(out) < len(reqs):
        most = max(most, len(st.active))
        for r, toks in st.step():
            out[owner[r.id]] = list(toks)
        if st.last_logits is not None:
            rs, lg = st.last_logits
            trace.append(([r.id for r in rs], lg.clone()))
        admit_all()
    return trace, out, most


@pytest.mark.parametrize("kind", ["bf16", "fp16", "nf4"])
def test_paged_stream_equals_contiguous_stream(model, ops, kind):
    V, cfg, sd = model
    eng = engine(model, kind)
    reqs = requests(cfg, eng.dtype, 8, seed=21)
    budgets = [9, 5, 7, 12, 6, 10, 4, 8]
    settings = mixed_settings(8)
    runs = []
    for pages in (None, 6 * 8):
        st = eng.decode_stream(6, max_positions=512, eos_token_id=-1, kv_pages=pages)
        try:
            runs.append(drive(st, reqs, budgets, settings))
        finally:
            st.close()
    (ta, oa, _), (tb, ob, _) = runs
    assert oa == ob
    assert len(ta) == len(tb)
    for (ia, la), (ib, lb) in zip(ta, tb):
        assert ia == ib and torch.equal(la, lb)


def test_paged_stream_holds_more_requests_in_the_same_bytes(model, ops):
    """2 contiguous slots of 512 rows hold the bytes of 24 pages of 64 k|v rows: the paged stream runs more than 2 requests at
    once, and in batch-invariant mode every answer equals the contiguous stream's"""
    from vstar_b200.kv_pages import PAGE_ROWS
    V, cfg, sd = model
    eng = engine(model, "bf16")
    S, Tm = 2, 512
    n_pages = S * Tm * 3 // (PAGE_ROWS * 2)
    reqs = requests(cfg, BF, 8, seed=23)
    budgets = [20, 40, 12, 30, 25, 8, 16, 35]
    greedy = [dict()] * 8
    lens = [eng.spliced_length(r[0], 0, r[3]) for r in reqs]
    with ops.batch_invariant():
        st = eng.decode_stream(S, max_positions=Tm, eos_token_id=-1)
        try:
            _, want, most_c = drive(st, reqs, budgets, greedy)
        finally:
            st.close()
        st = eng.decode_stream(8, max_positions=Tm, eos_token_id=-1, kv_pages=n_pages)
        try:
            assert st._cache.numel() * st._cache.element_size() == S * Tm * 3 * cfg.hidden * 2 * cfg.n_layers
            _, got, most_p = drive(st, reqs, budgets, greedy, fits=lambda i: st.pages.need(lens[i], budgets[i]) <= st.pages.free_pages)
            st.pages.check()
        finally:
            st.close()
    assert most_c == S and most_p > S, (most_c, most_p)
    assert got == want


def _requested():
    return torch.cuda.memory_stats()["requested_bytes.all.current"]


def test_paged_stream_device_memory_is_pool_scratch_and_table(model, ops):
    """the bytes the stream requests are its pool, scratch and page table (memory_allocated counts the caching allocator's
    blocks, which may be larger than the request when a cached block is reused unsplit)"""
    V, cfg, sd = model
    eng = engine(model, "bf16")
    reqs = requests(cfg, BF, 2)
    eng.decode_stream(1, max_positions=64, kv_pages=1).close()                     # builds the layer table once
    gc.collect()
    torch.cuda.synchronize()
    m0, r0 = torch.cuda.memory_allocated(), _requested()
    slots, Tm, N, c = 3, 512, 20, cfg
    st = eng.decode_stream(slots, max_positions=Tm, eos_token_id=-1, kv_pages=N)
    pool = c.n_layers * N * 64 * 2 * c.hidden * 2
    scratch = slots * (5 * c.hidden + c.intermediate) * 2
    table = slots * (Tm // 64) * 4
    assert _requested() - r0 == pool + scratch + table
    assert torch.cuda.memory_allocated() - m0 >= pool + scratch + table
    torch.cuda.reset_peak_memory_stats()
    for r in reqs:
        st.admit(r, 4)
    while st.active:
        st.step()
    assert st.pages.free_pages == N
    st.close()
    del st
    gc.collect()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == m0


def test_paged_free_form_inference_stream_equals_contiguous(model, ops):
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
        want = dict(llm.free_form_inference_stream(items, max_new_tokens=6, slots=2))
        got = dict(llm.free_form_inference_stream(items, max_new_tokens=6, slots=4, kv_pages=12))
        beams = dict(llm.free_form_inference_stream(items, max_new_tokens=6, slots=4, num_beams=2))
        beams_paged = dict(llm.free_form_inference_stream(items, max_new_tokens=6, slots=4, num_beams=2, kv_pages=16))
    assert got == want and beams_paged == beams
