"""Growing paged decode stream (DecodeStream(kv_pages=N, kv_swap_pages=M)): pages taken as rows are written, requests swapped
to pinned host memory when the pool runs dry.

(1) vsb_swap_pages_b16 out and back in, into other pages, restores every bit (bf16 / fp16, P = 16 / 64, the pool's first and
    last pages, lists longer than one launch, a 7B-shaped page) and refuses bad arguments before any launch;
(2) in batch-invariant mode, greedy, sampled and beam (k = 2, 4) requests with 512-token budgets on a pool too small for their
    reservations are preempted, and still give the tokens, beam scores and bit-identical logits of a reserve-ahead stream
    that never binds, in bf16, fp16 and NF4;
(3) when the pool never binds, the growing stream admits, steps and emits exactly what the reserve-ahead stream does, with
    bit-identical logits in default mode;
(4) in the bytes of S contiguous slots, the growing stream decodes more requests at once than the reserve-ahead one when the
    answers end well before their budgets;
(5) device memory returns to its level before the stream, and close() frees the swap area;
(6) free_form_inference_stream(kv_pages=N, kv_swap_pages=M) equals the call without swap, in batch-invariant mode."""
import gc
import weakref

import numpy as np
import pytest
import torch

from tests.test_vqa_stream_gpu import bits, engine, model, ops, randn, requests  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu
BF, F16 = torch.bfloat16, torch.float16


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("dt", [BF, F16])
@pytest.mark.parametrize("L,N,P,W,M,n", [
    (2, 12, 16, 64, 9, 7),
    (3, 10, 64, 96, 10, 10),
    (2, 900, 16, 64, 800, 777),          # three launches of VSB_SWAP_PAGES_PER_LAUNCH pairs
    (4, 6, 64, 8192, 5, 5),              # a 7B k|v page
])
def test_swap_out_and_in_restores_every_bit(ops, dt, L, N, P, W, M, n):
    g = torch.Generator().manual_seed(N + P + W)
    pool = randn(L, N, P, W, seed=N + W).to(dt).cuda()
    want = pool.clone()
    host = torch.full((M, L, P, W), float("nan"), dtype=dt).pin_memory()
    mid = [p for p in torch.randperm(N, generator=g).tolist() if p not in (0, N - 1)][:n - 2]
    src = [0] + mid + [N - 1]                                                   # the pool's first and last page
    assert len(set(src)) == n
    slots = torch.randperm(M, generator=g)[:n].tolist()
    ops.swap_pages(pool, host, list(zip(src, slots)), to_host=True)
    torch.cuda.synchronize()
    for p, s in zip(src, slots):
        assert torch.equal(bits(host[s]), bits(want[:, p].cpu()))
    dst = torch.randperm(N, generator=g)[:n].tolist()
    pool.fill_(float("nan"))
    ops.swap_pages(pool, host, list(zip(dst, slots)), to_host=False)
    torch.cuda.synchronize()
    for p, q in zip(dst, src):
        assert torch.equal(bits(pool[:, p]), bits(want[:, q]))
    untouched = sorted(set(range(N)) - set(dst))
    if untouched:
        assert torch.isnan(pool[:, untouched].float()).all()


def test_swap_pages_refuses_bad_arguments(ops):
    from vstar_b200 import _lib
    L, N, P, W, M = 2, 8, 16, 64, 4
    pool = torch.zeros((L, N, P, W), dtype=BF, device="cuda")
    host = torch.zeros((M, L, P, W), dtype=BF).pin_memory()
    bad = [([(N, 0)], True), ([(-1, 0)], False), ([(0, M)], True), ([(0, 1), (1, 1)], True), ([(2, 0), (2, 1)], False)]
    for pairs, out in bad:
        with pytest.raises(_lib.VsbError):
            ops.swap_pages(pool, host, pairs, to_host=out)
    with pytest.raises(_lib.VsbError):
        ops.swap_pages(pool, torch.zeros((M, L, P, W), dtype=BF), [(0, 0)], to_host=True)     # not pinned
    with pytest.raises(_lib.VsbError):
        _lib.call("vsb_swap_pages_b16", pool.data_ptr(), L, pool.stride(0), N, pool.stride(1), P * W, None, M, host.stride(0),
                  host.stride(1), (_lib.ctypes.c_int * 1)(0), (_lib.ctypes.c_int * 1)(0), 1, 1, None)
    ops.swap_pages(pool, host, [(1, 0), (0, 1)], to_host=False)                 # two pages from two slots is fine
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ streams
def make_stream(eng, slots, positions, kv_pages, kv_swap_pages=None, ends=None):
    from vstar_b200.vqa import DecodeStream

    class EndsAt(DecodeStream):
        """request i ends after ends[i] tokens, standing in for a trained model's eos"""
        def _ended(self, r):
            return (ends is not None and len(r.tokens) >= ends[r.id]) or super()._ended(r)

    return EndsAt(eng, slots, positions, -1, kv_pages=kv_pages, kv_swap_pages=kv_swap_pages)


def drive(st, reqs, budgets, settings, lens):
    """admit in order whenever the stream's rule allows -> ({index: [logits rows of each call it took part in]}, {index: handle},
    trace of (ids, logits) per call, most requests decoding at once)"""
    rows, handles, trace, nxt, most = {}, {}, [], 0, 0

    def fits():
        k = settings[nxt].get("num_beams", 1)
        free = st.free_rows(k)
        if free is None:
            return False
        if st.growing:
            return st.pages.can_admit(free, lens[nxt], budgets[nxt])
        return st.pages.need(lens[nxt], budgets[nxt], k) <= st.pages.free_pages

    def record():
        rs, lg = st.last_logits
        trace.append(([r.id for r in rs], lg.clone()))
        at = {}
        for i, r in enumerate(rs):
            at.setdefault(r.id, []).append(i)
        for rid, idx in at.items():
            rows.setdefault(rid, []).append(lg[idx].clone())

    def admit_all():
        nonlocal nxt
        while nxt < len(reqs) and fits():
            h = st.admit(reqs[nxt], budgets[nxt], **settings[nxt])
            assert h.id == nxt
            handles[nxt] = h
            record()
            nxt += 1
    admit_all()
    while nxt < len(reqs) or any(not h.done for h in handles.values()):
        most = max(most, len(st.active))
        before = st.steps
        st.step()
        if st.steps > before:
            record()
        if st.growing:
            st.pages.check()
        admit_all()
    return rows, handles, trace, most


SETTINGS = [dict(), dict(temperature=0.8, top_k=20, top_p=0.9, seed=11), dict(), dict(num_beams=2), dict(temperature=1.1, seed=-5),
            dict(num_beams=4), dict(), dict(num_beams=2)]


@pytest.mark.parametrize("kind", ["bf16", "fp16", "nf4"])
def test_preempted_requests_keep_their_logits(model, ops, kind):
    V, cfg, sd = model
    eng = engine(model, kind)
    n = len(SETTINGS)
    reqs = requests(cfg, eng.dtype, n, seed=31)
    lens = [eng.spliced_length(r[0], 0, r[3]) for r in reqs]
    budgets = [512] * n
    positions = max(lens) + 512
    from vstar_b200.kv_pages import PagePool
    sizer = PagePool(1, 1, 1)
    fulls = [sizer.need(T, 512, s.get("num_beams", 1)) for T, s in zip(lens, SETTINGS)]
    runs = []
    with ops.batch_invariant():
        for pages, swap in ((sum(fulls), None), (max(fulls) + 4, 4 * sum(fulls))):
            st = make_stream(eng, 16, positions, pages, swap)
            try:
                runs.append(drive(st, reqs, budgets, SETTINGS, lens) + (st.preemptions, st.swapped_pages, st.restored_pages))
            finally:
                st.close()
    (ra, ha, _, _, pa, _, _), (rb, hb, _, _, pb, out, back) = runs
    assert pa == 0 and pb > 0 and out == back > 0
    assert any(h.preemptions and h.kind == "beam" for h in hb.values())
    assert sum(h.preemptions for h in hb.values()) == pb
    for i in range(n):
        assert ha[i].tokens == hb[i].tokens, i
        assert ha[i].score == hb[i].score, i
        assert len(ra[i]) == len(rb[i]), i
        for a, b in zip(ra[i], rb[i]):
            assert torch.equal(a, b), i


def test_growing_stream_equals_reserve_ahead_when_the_pool_never_binds(model, ops):
    V, cfg, sd = model
    eng = engine(model, "bf16")
    reqs = requests(cfg, BF, 8, seed=21)
    lens = [eng.spliced_length(r[0], 0, r[3]) for r in reqs]
    budgets = [9, 5, 70, 12, 6, 10, 4, 8]
    runs = []
    for swap in (None, 64):
        st = make_stream(eng, 6, 512, 200, swap)
        try:
            runs.append(drive(st, reqs, budgets, SETTINGS, lens))
            assert st.preemptions == 0
        finally:
            st.close()
    (_, ha, ta, _), (_, hb, tb, _) = runs
    assert [h.tokens for h in ha.values()] == [h.tokens for h in hb.values()]
    assert len(ta) == len(tb)
    for (ia, la), (ib, lb) in zip(ta, tb):
        assert ia == ib and torch.equal(la, lb)


def test_growing_stream_holds_more_requests_in_the_same_bytes(model, ops):
    """2 contiguous slots of 1024 rows hold the bytes of 48 pages; with 512-token budgets and answers of 10-40 tokens the
    growing stream decodes more requests at once than the reserve-ahead one, with the same answers"""
    from vstar_b200.kv_pages import PAGE_ROWS
    V, cfg, sd = model
    eng = engine(model, "bf16")
    S, Tm = 2, 1024
    n_pages = S * Tm * 3 // (PAGE_ROWS * 2)
    n = 12
    reqs = requests(cfg, BF, n, seed=23)
    lens = [eng.spliced_length(r[0], 0, r[3]) for r in reqs]
    ends = [10 + (7 * i) % 31 for i in range(n)]
    greedy, budgets = [dict()] * n, [512] * n
    out = []
    with ops.batch_invariant():
        for swap in (None, 4 * n_pages):
            st = make_stream(eng, n, Tm, n_pages, swap, ends=ends)
            try:
                _, h, _, most = drive(st, reqs, budgets, greedy, lens)
                out.append(([h[i].tokens for i in range(n)], most, st.occupied / st.steps))
            finally:
                st.close()
    (ta, most_r, occ_r), (tb, most_g, occ_g) = out
    assert ta == tb
    assert most_g > most_r and occ_g > occ_r, (most_r, most_g, occ_r, occ_g)


def test_growing_stream_frees_device_memory_and_the_swap_area(model, ops):
    V, cfg, sd = model
    eng = engine(model, "bf16")
    reqs = requests(cfg, BF, 3)
    make_stream(eng, 1, 64, 1).close()                                          # builds the layer table once
    gc.collect()
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    st = make_stream(eng, 4, 512, 20, 40)
    assert st._swap.is_pinned() and tuple(st._swap.shape) == (40, cfg.n_layers, 64, 2 * cfg.hidden)
    for r in reqs:
        st.admit(r, 70)
    while st.active:
        st.step()
    assert st.pages.free_pages == 20 and st.pages.free_swap_pages == 40
    swap = weakref.ref(st._swap)
    st.close()
    del st
    gc.collect()
    torch.cuda.synchronize()
    assert swap() is None
    assert torch.cuda.memory_allocated() == m0


def test_growing_free_form_inference_stream_equals_reserve_ahead(model, ops):
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
        want = dict(llm.free_form_inference_stream(items, max_new_tokens=80, slots=4, kv_pages=40))
        got = dict(llm.free_form_inference_stream(items, max_new_tokens=80, slots=4, kv_pages=12, kv_swap_pages=64))
        beams = dict(llm.free_form_inference_stream(items, max_new_tokens=80, slots=4, num_beams=2, kv_pages=40))
        beams_swap = dict(llm.free_form_inference_stream(items, max_new_tokens=80, slots=4, num_beams=2, kv_pages=16, kv_swap_pages=64))
    assert got == want and beams_swap == beams
    with pytest.raises(ValueError, match="kv_swap_pages"):
        dict(llm.free_form_inference_stream(items, max_new_tokens=80, slots=4, kv_pages=40, kv_swap_pages=1))
