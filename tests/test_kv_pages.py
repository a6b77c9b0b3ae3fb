"""Page allocator of the paged decode stream (vstar_b200.kv_pages), without a GPU:
(1) reservations of greedy / sampled and beam requests, at prompts that end on a page boundary and one row before it;
(2) reference counts of shared prompt pages, release when a request ends and when the stream closes;
(3) DecodeStream(kv_pages=N).admit refuses short pages or slots before anything reaches the device;
(4) a randomised admit / fork / end sequence never gives a page to two owners and leaves the pool whole."""
import random

import numpy as np
import pytest

from tests.test_stream_modes import HostEngine
from vstar_b200 import _lib
from vstar_b200.beam import fork_slots
from vstar_b200.kv_pages import PAGE_ROWS, PagePool, pages_for
from vstar_b200.vqa import DecodeStream

P = PAGE_ROWS


def test_page_rows_is_a_power_of_two():
    assert P == 64 and P & (P - 1) == 0
    with pytest.raises(ValueError):
        PagePool(4, 2, 2, page_rows=48)
    with pytest.raises(ValueError):
        PagePool(4, 2, 2, page_rows=8)
    with pytest.raises(ValueError):
        PagePool(0, 2, 2)


@pytest.mark.parametrize("T,n,want", [
    (2 * P, 1, 3), (2 * P - 1, 1, 2), (2 * P - 1, 2, 3), (2 * P, P, 3), (2 * P - 1, P + 1, 3), (1, 1, 1), (600, 200, 13)])
def test_single_row_reserves_prompt_plus_budget(T, n, want):
    pool = PagePool(40, 4, 32)
    assert pool.need(T, n) == want == pages_for(T + n)
    assert pool.reserve([2], T, n) == 0
    pages = pool.owned[2]
    assert len(pages) == want and len(set(pages)) == want
    assert pool.table[2, :want].tolist() == pages and not pool.table[2, want:].any()
    assert pool.free_pages == 40 - want and all(pool.refs[p] == 1 for p in pages)
    pool.check()


@pytest.mark.parametrize("T", [3 * P, 3 * P - 1, 3 * P + 1, P - 1])
@pytest.mark.parametrize("k", [2, 4])
def test_beams_share_the_full_prompt_pages(T, k):
    n = 100
    pool = PagePool(64, 8, 16)
    rows = [5, 1, 6, 0][:k]
    full, shared = pages_for(T + n), T // P
    assert pool.need(T, n, k) == shared + k * (full - shared)
    assert pool.reserve(rows, T, n) == shared
    common = pool.owned[rows[0]][:shared]
    for r in rows:
        pages = pool.owned[r]
        assert len(pages) == full and pages[:shared] == common
        assert all(pool.refs[p] == k for p in pages[:shared]) and all(pool.refs[p] == 1 for p in pages[shared:])
    private = [p for r in rows for p in pool.owned[r][shared:]]
    assert len(set(private)) == len(private) and not set(private) & set(common)
    assert pool.free_pages == 64 - pool.need(T, n, k)
    # a beam that dies leaves the shared pages to the others; the last one returns them
    pool.release(rows[:1])
    assert all(pool.refs[p] == k - 1 for p in common)
    pool.check()
    pool.release(rows[1:])
    assert pool.free_pages == 64 and not any(pool.refs) and not pool.table.any()
    pool.check()


def test_refusals_change_nothing():
    pool = PagePool(9, 3, 8)
    pool.reserve([0], 2 * P, P)                                  # 3 pages
    before = (list(pool.refs), pool.free_pages, pool.table.copy())
    with pytest.raises(RuntimeError, match="in use"):
        pool.reserve([0], 10, 10)
    with pytest.raises(RuntimeError, match="pages of a page-table row"):
        pool.reserve([1], 8 * P, 1)
    with pytest.raises(RuntimeError, match="not enough free KV pages"):
        pool.reserve([1, 2], 3 * P + 1, P)                       # 3 shared + 2 x 2 private > 6 free
    assert (list(pool.refs), pool.free_pages) == before[:2] and np.array_equal(pool.table, before[2])
    pool.release_all()
    assert pool.free_pages == 9
    pool.check()


def test_random_admit_fork_end_sequences_keep_the_pool_whole():
    rng = random.Random(0)
    for trial in range(30):
        n_pages, rows = rng.randint(8, 60), rng.randint(2, 12)
        pool = PagePool(n_pages, rows, 12)
        running = []                                             # page-table rows of each running request
        for _ in range(200):
            op = rng.random()
            free_rows = [r for r in range(rows) if pool.owned[r] is None]
            if op < 0.5 and free_rows:
                k = rng.choice([1, 1, 2, 4])
                T, n = rng.randint(1, 8 * P), rng.randint(1, 3 * P)
                want = rng.sample(free_rows, min(k, len(free_rows)))
                if pages_for(T + n) > 12:
                    continue
                try:
                    pool.reserve(want, T, n)
                    running.append((want, T))
                except RuntimeError:
                    assert pool.need(T, n, len(want)) > pool.free_pages
            elif op < 0.7 and running:
                # a beam fork copies the parent's generated rows [T, ...) into the child's pages: those pages are the child's
                # alone and none of them is one the parent reads
                req, T = rng.choice(running)
                old = rng.sample(req, len(req))
                _, forks = fork_slots(old, [(0.0, 0, rng.randrange(len(req))) for _ in req], req)
                for src, dst in forks:
                    written = pool.owned[dst][T // P:]
                    assert all(pool.refs[p] == 1 for p in written) and not set(written) & set(pool.owned[src])
            elif running:
                pool.release(running.pop(rng.randrange(len(running)))[0])
            pool.check()
            owners = {}
            for req_i, (req, _) in enumerate(running):
                for r in req:
                    for p in set(pool.owned[r]):
                        assert owners.setdefault(p, req_i) == req_i, "a page owned by two requests"
        for req, _ in running:
            pool.release(req)
        assert pool.free_pages == n_pages and not any(pool.refs)
        pool.check()


# ------------------------------------------------------------------------------------------------ the stream's admission
def paged_host_stream(n_pages, max_slots=4, busy=(), max_positions=8 * P):
    st = DecodeStream.__new__(DecodeStream)
    st.engine, st.eos = HostEngine(), 2
    st.max_slots, st.max_positions = max_slots, max_positions
    st._cache = object()                                         # open; admit must raise before it is touched
    st._slots = [None] * max_slots
    st.pages = PagePool(n_pages, max_slots, pages_for(max_positions))
    for r in busy:
        st._slots[r] = object()
        st.pages.reserve([r], P, 1)
    return st


@pytest.mark.parametrize("T,n,kw,exc,match", [
    (3 * P, P, {}, RuntimeError, "not enough free KV pages"),            # 4 pages, 3 free
    (P, 2, dict(num_beams=4), RuntimeError, "no free slot"),             # 2 of 4 slots free
    (3 * P - 1, 2, dict(num_beams=2), RuntimeError, "not enough free KV pages"),     # 2 shared + 2 x 2 private > 3
    (8 * P - 3, 4, {}, _lib.VsbError, "exceeds"),                        # past max_positions
    (P, 2, dict(num_beams=5), ValueError, "slots"),
])
def test_paged_admit_refuses_before_any_launch(T, n, kw, exc, match):
    st = paged_host_stream(7, busy=[0, 3])                       # 2 pages each
    free0 = st.pages.free_pages
    n0 = _lib.launches
    with pytest.raises(exc, match=match):
        st.admit(([1] * T, None, None, None, None), n, **kw)
    assert _lib.launches == n0 and st.pages.free_pages == free0
    st.pages.check()


def test_paged_admit_that_fits_reaches_the_device():
    """the checks pass: admission goes on to embed the prompt (here the host engine has no device, so it stops there)"""
    st = paged_host_stream(8, busy=[0])
    with pytest.raises(AttributeError, match="build_embeds"):
        st.admit(([1] * (3 * P - 1), None, None, None, None), 2, num_beams=2)       # 2 shared + 2 x 2 private = 6 pages
    assert st.pages.free_pages == 6                              # nothing reserved before the prefill


def test_paged_release_on_end_and_close():
    st = paged_host_stream(12)
    from vstar_b200.vqa import StreamRequest
    r = StreamRequest(0, 1, 2 * P, 10, None, slots=[1, 2])
    st.pages.reserve([1, 2], 2 * P, 10)
    st._slots[1] = st._slots[2] = r
    assert st.pages.free_pages == 12 - 4
    st._release(r)
    assert r.done and st.pages.free_pages == 12 and st.free_slots == 4
    st.pages.reserve([0], P, 1)
    st.pages.reserve([3], P, 1)
    st._scratch = st._deq = None
    st.close()
    assert st.pages.free_pages == 12
    st.pages.check()
