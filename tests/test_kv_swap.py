"""Growing page pool with swap (vstar_b200.kv_pages.GrowingPool, DecodeStream(kv_pages=N, kv_swap_pages=M)), without a GPU:
(1) admission takes the prompt's pages (beams share the full ones), growth appends a page when a row reaches a page's first row;
(2) victims are the newest running requests, and preempted requests resume oldest first, shared pages swapped once and shared
    again after resumption;
(3) randomised admit / step / preempt / resume / end sequences of greedy and beam requests keep check() true, every request
    finishes when the pool holds exactly the largest one, and release_all frees every page and swap slot;
(4) refusals are raised before any state changes."""
import copy
import random

import pytest

from tests.test_stream_modes import HostEngine
from vstar_b200 import _lib
from vstar_b200.kv_pages import PAGE_ROWS, GrowingPool, pages_for
from vstar_b200.vqa import DecodeStream

P = PAGE_ROWS


def state(pool):
    return copy.deepcopy({k: v.tolist() if k == "table" else v for k, v in vars(pool).items()})


@pytest.mark.parametrize("T", [2 * P, 2 * P + 1, 2 * P - 1])
@pytest.mark.parametrize("k", [1, 2, 5])
def test_admission_takes_the_prompt_pages_and_growth_follows_writes(T, k):
    pool = GrowingPool(64, 8, 16, 64)
    rows = [6, 1, 3, 0, 7][:k]
    shared = pool.admit("a", rows, T, 300)
    assert shared == (T // P if k > 1 else 0)
    for r in rows:
        assert len(pool.owned[r]) == pages_for(T)
        assert pool.owned[r][:shared] == pool.owned[rows[0]][:shared]
    assert pool.free_pages == 64 - pool.need(T, 0, k)
    n = 0
    for step in range(2 * P + 3):
        before = pool.free_pages
        pos = pool.pos["a"]
        resumed, preempted, changed = pool.schedule()
        assert not resumed and not preempted
        grew = pos % P == 0
        assert changed == grew and pool.free_pages == before - (k if grew else 0)
        for r in rows:
            assert len(pool.owned[r]) == pos // P + 1 == pages_for(pos + 1)
        n += grew
        pool.check()
    pool.finish("a")
    assert pool.free_pages == 64
    pool.check()


def test_victims_newest_first_and_resume_oldest_first():
    pool = GrowingPool(8, 6, 8, 64)
    for key, row in zip("abcd", range(4)):
        pool.admit(key, [row], P - 1, 4 * P)                 # one page each; each grows at its next write
    assert pool.free_pages == 4 and pool.growth() == 0
    pool.schedule()                         # writes row P - 1
    assert pool.growth() == 4
    pool.schedule()                         # the four pages fit: every request now holds two
    assert pool.free_pages == 0 and pool.growth() == 0
    for _ in range(P - 1):
        pool.schedule()
    assert pool.growth() == 4                                 # all four reach their third page at once
    resumed, preempted, _ = pool.schedule()
    assert [k for k, _ in preempted] == ["d", "c"] and not resumed
    assert pool.preempted == ["d", "c"] and pool.running == ["a", "b"]
    assert pool.free_pages == 2 and pool.free_swap_pages == 64 - 4
    pool.check()
    with pytest.raises(RuntimeError, match="wait to resume"):
        pool.check_admit([4], 1, 1)
    pool.finish("b")                                          # five pages free: d (2 pages + 1 growth) comes back first, c does not fit
    resumed, preempted, _ = pool.schedule()
    assert [k for k, _, _ in resumed] == ["d"] and not preempted
    assert pool.running == ["a", "d"] and pool.preempted == ["c"]
    pool.check()
    pool.finish("a")
    resumed, _, _ = pool.schedule()
    assert [k for k, _, _ in resumed] == ["c"] and pool.running == ["d", "c"]
    # the newest is now the resumed c
    assert pool.running[-1] == "c"
    pool.check()


@pytest.mark.parametrize("T", [2 * P, 2 * P + 1])
def test_shared_prompt_pages_swap_once_and_share_again(T):
    k = 4
    pool = GrowingPool(64, 8, 8, 64)
    pool.admit("old", [0], 10, 10)
    pool.admit("beam", [1, 2, 3, 4], T, 100)
    shared = T // P
    held = {p for r in (1, 2, 3, 4) for p in pool.owned[r]}
    pairs = pool.swap_out("beam")
    assert sorted(p for p, _ in pairs) == sorted(held) and len(pairs) == shared + k * (pages_for(T) - shared)
    assert pool.free_swap_pages == 64 - len(pairs)
    pool.check()
    rows = [7, 5, 6, 1]
    back = pool.swap_in("beam", rows)
    assert sorted(s for s, _ in back) == sorted(s for _, s in pairs)
    common = pool.owned[rows[0]][:shared]
    for r in rows:
        assert pool.owned[r][:shared] == common
        assert pool.table[r, :len(pool.owned[r])].tolist() == pool.owned[r]
    assert all(pool.refs[p] == k for p in common)
    assert pool.free_swap_pages == 64
    pool.check()


def run(pool, reqs, check=True):
    """admit (in order, by the pool's rule) and step the requests [(prompt rows, beams, answer length, budget)] until all end
    -> the order they resumed and were preempted in"""
    nxt, live, log = 0, {}, []
    while nxt < len(reqs) or live or pool.preempted:
        while nxt < len(reqs):
            T, k, n, budget = reqs[nxt]
            rows = pool.free_rows(k)
            if rows is None or not pool.can_admit(rows, T, budget):
                break
            pool.admit(nxt, rows, T, budget)
            live[nxt] = n
            if n == 1:                                        # ended at admission on the prefill's token
                pool.finish(nxt)
                del live[nxt]
            nxt += 1
            if check:
                pool.check()
        resumed, preempted, changed = pool.schedule()
        log.append(([k for k, _ in preempted], [k for k, _, _ in resumed]))
        if check:
            pool.check()
        for key in list(pool.running):
            for r in pool.rows_of[key]:
                assert pool.pos[key] - 1 < len(pool.owned[r]) * P    # the row the step wrote has its page
            if pool.pos[key] - reqs[key][0] + 1 >= live[key]:       # its last token came from this step
                pool.finish(key)
                del live[key]
                if check:
                    pool.check()
    return log


@pytest.mark.parametrize("seed", range(12))
def test_random_streams_keep_the_pool_whole(seed):
    rng = random.Random(seed)
    reqs = []
    for _ in range(rng.randint(6, 20)):
        k = rng.choice([1, 1, 1, 2, 4, 8, 16])
        T = rng.choice([P, 2 * P, 2 * P + 1, 3 * P - 1, rng.randint(1, 4 * P)])
        budget = rng.randint(1, 4 * P)
        reqs.append((T, k, rng.randint(1, budget), budget))
    rows = 24
    largest = max(GrowingPool(1, 1, 1, 1).need(T, b, k) for T, k, _, b in reqs)
    pool = GrowingPool(largest + rng.randint(0, 8), rows, 8, largest * rng.randint(1, 4))
    log = run(pool, reqs)
    victims = [v for out, _ in log for v in out]
    resumes = [v for _, back in log for v in back]
    assert sorted(victims) == sorted(resumes)                  # everything preempted came back
    assert pool.free_pages == pool.n_pages and pool.free_swap_pages == pool.swap_pages
    pool.check()


def test_a_pool_of_exactly_the_largest_request_finishes_and_preempts():
    reqs = [(P - 1, 1, 3 * P, 3 * P), (P, 4, 2 * P, 2 * P), (3, 1, 4 * P, 4 * P), (2 * P + 1, 2, P, 2 * P), (5, 1, 2, 2)]
    largest = max(GrowingPool(1, 1, 1, 1).need(T, b, k) for T, k, _, b in reqs)
    pool = GrowingPool(largest, 16, 8, 4 * largest)
    log = run(pool, reqs)
    assert any(out for out, _ in log)                          # the small pool had to preempt
    assert pool.free_pages == largest and not pool.running and not pool.preempted
    pool.check()


def test_release_all_frees_pages_and_swap_slots():
    pool = GrowingPool(16, 8, 8, 32)
    pool.admit(0, [0], 3 * P, 10)
    pool.admit(1, [1, 2], 2 * P + 1, 10)
    pool.swap_out(1)
    pool.release_all()
    assert pool.free_pages == 16 and pool.free_swap_pages == 32 and not pool.running and not pool.preempted
    assert not pool.table.any()
    pool.check()


def two_running():
    pool = GrowingPool(10, 8, 16, 8)
    pool.admit(0, [0], 3 * P, P)                                         # 3 pages now, 4 at full length; grows next step
    pool.admit(1, [1], P - 1, 2)                                         # 1 page
    return pool


@pytest.mark.parametrize("args,match", [
    (([0], 10, 10), "in use"),
    (([5], 10 * P, 10), "exceed"),                                       # 11 pages > the pool of 10
    (([5], 5 * P, 10), "not enough free KV pages"),                      # 5 + its growth 1 + the running growth 1 > 6 free
    (([5], 10, 6 * P), "swap area"),                                     # full lengths 4 + 1 + 7 less the smallest > 8
])
def test_admit_refusals_change_nothing(args, match):
    pool = two_running()
    before = state(pool)
    with pytest.raises(RuntimeError, match=match):
        pool.admit(9, *args)
    assert state(pool) == before and not pool.can_admit(*args)
    pool.check()


@pytest.mark.parametrize("call,match", [
    (lambda p: p.admit(9, [5], 1, 1), "wait to resume"),
    (lambda p: p.swap_in(0, [5]), "not the next to resume"),
    (lambda p: p.swap_in(2, [5, 6]), "not 1 free rows"),
    (lambda p: p.swap_in(2, [0]), "not 1 free rows"),
])
def test_resume_refusals_change_nothing(call, match):
    pool = two_running()
    pool.admit(2, [2], 2 * P + 4, 1)                                     # 3 pages
    pool.swap_out(2)
    before = state(pool)
    with pytest.raises(RuntimeError, match=match):
        call(pool)
    assert state(pool) == before
    pool.check()


def test_swap_out_beyond_the_swap_area_changes_nothing():
    pool = GrowingPool(10, 8, 16, 2)
    pool.admit(0, [0], 3 * P, 1)
    before = state(pool)
    with pytest.raises(RuntimeError, match="swap area"):
        pool.swap_out(0)
    assert state(pool) == before


def test_growth_past_the_free_pages_changes_nothing():
    pool = GrowingPool(3, 4, 4, 8)
    pool.admit(0, [0], P, 2)
    pool.admit(1, [1], P - 1, 2)
    pool.grow()                                               # request 0's page for row P; request 1 reaches row P next
    pool.pos[0] += 1
    pool.pos[1] += 1
    before = state(pool)
    with pytest.raises(RuntimeError, match="new pages"):
        pool.grow()
    assert state(pool) == before


def test_pool_refuses_an_empty_swap_area():
    with pytest.raises(ValueError):
        GrowingPool(4, 2, 2, 0)


def test_stream_refuses_swap_pages_without_kv_pages():
    n0 = _lib.launches
    with pytest.raises(ValueError, match="kv_pages"):
        DecodeStream(HostEngine(), 2, 100, kv_swap_pages=4)
    assert _lib.launches == n0


def growing_host_stream(n_pages, swap, busy=(), max_slots=4, max_positions=8 * P):
    st = DecodeStream.__new__(DecodeStream)
    st.engine, st.eos = HostEngine(), 2
    st.max_slots, st.max_positions = max_slots, max_positions
    st._cache = object()
    st.pages = GrowingPool(n_pages, max_slots, pages_for(max_positions), swap)
    st._slots = [None] * max_slots
    for i, s in enumerate(busy):
        st.pages.admit(100 + i, [s], 2 * P - 1, 2)
        st._slots[s] = object()
    return st


@pytest.mark.parametrize("T,n,kw,match", [
    (3 * P, 1, {}, "not enough free KV pages"),               # 3 pages + 1 growth > 3 free
    (2 * P, 4 * P, {}, "swap area"),                          # full length 6 pages besides the smaller live one > 4
    (P - 1, 2, dict(num_beams=3), "no free slot"),
])
def test_growing_admit_refuses_before_any_launch(T, n, kw, match):
    st = growing_host_stream(7, 4, busy=[0, 3])               # 2 pages each
    before = state(st.pages)
    n0 = _lib.launches
    with pytest.raises(RuntimeError, match=match):
        st.admit(([1] * T, None, None, None, None), n, **kw)
    assert _lib.launches == n0 and state(st.pages) == before


def test_growing_admit_that_fits_reaches_the_device():
    st = growing_host_stream(7, 8, busy=[0])
    with pytest.raises(AttributeError, match="build_embeds"):
        st.admit(([1] * (2 * P - 1), None, None, None, None), 2, num_beams=2)    # 1 shared + 2 x 1 private
    assert st.pages.free_pages == 5                           # nothing taken before the prefill


def test_seal_passes_kv_swap_pages_on_only_when_set(monkeypatch):
    """python -m vstar_b200.seal --kv-pages N --kv-swap-pages M reaches free_form_inference_stream; without the flags the call
    carries neither keyword, so a VQA LLM with the older signature keeps working"""
    from tests.test_seal_open import OpenStubLLM, StubVSM
    from tests import seal_open_helpers as H
    from vstar_b200 import seal
    from vstar_b200 import visual_search as VS

    def stream(self, states, window=None):
        for st in states:
            yield st, H.fake_search(st.target, st.image)
    monkeypatch.setattr(VS.SearchController, "stream", stream)
    seen = []

    class Recording(OpenStubLLM):
        def free_form_inference_stream(self, items, max_new_tokens=200, slots=16, **kw):
            seen.append(kw)
            return super().free_form_inference_stream(items, max_new_tokens, slots)

    a = seal.build_parser().parse_args(["--image", "x.png", "--question", "q", "--kv-pages", "40", "--kv-swap-pages", "90"])
    assert (a.kv_pages, a.kv_swap_pages) == (40, 90)
    items = [(H.case_image(c), c[0]) for c in H.CASES[:3]]
    want = seal.answer_open_many(Recording(), StubVSM(), items)
    assert seen and all(kw == {} for kw in seen)
    seen.clear()
    got = seal.answer_open_many(Recording(), StubVSM(), items, kv_pages=40, kv_swap_pages=90)
    assert seen and all(kw == dict(kv_pages=40, kv_swap_pages=90) for kw in seen)
    assert [o[0] for o in got] == [o[0] for o in want]
