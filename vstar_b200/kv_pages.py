"""Page allocator of the paged decode stream (DecodeStream(kv_pages=N)), pure host code.

The pool holds N pages of PAGE_ROWS k|v rows per layer.  A decode row (a greedy or sampled request, or one beam of a beam
request) owns one row of the page table: the pages that hold its keys, in order, so key j sits in page table[row][j // P] at
row j % P.  Pages are reserved at admission for the whole request, prompt plus max_new_tokens, and never grow or move while it
runs; they return to the pool when it ends or the stream closes.

A beam request of k beams shares the full pages of its prompt among its beams (a reference count per page) and gives every beam
private pages from the prompt's last, partly filled page on: the beams write their generated rows there, and a fork copies the
parent's generated rows into the child's private pages, so no page a step writes is shared.

GrowingPool (DecodeStream(kv_pages=N, kv_swap_pages=M)) takes pages on demand instead: a request takes the pages its prompt
fills at admission and one more page per row whenever a step is about to write a page's first row.  When the free pages cannot
cover a step's growth, the newest running request (by admission or resumption) is preempted: its pages are copied to a swap area
of M host pages (each shared prompt page once) and freed, and it resumes, oldest preempted first and before any new admission,
into whichever pages and page-table rows are free, with its sharing restored.
"""
from __future__ import annotations

import numpy as np

PAGE_ROWS = 64                                   # rows per page: a power of two >= 16 (the kernels' page_rows)


def pages_for(rows, page_rows=PAGE_ROWS):
    return -(-int(rows) // page_rows)


def plan_chunks(pending, budget):
    """the prompt rows one step of a chunked-prefill stream (DecodeStream(prefill_chunk=C)) carries: pending = [(request,
    rows written, prompt rows)] of the requests still prefilling, in admission order; budget = C.  -> [(request, first row,
    rows)], at most `budget` rows in all, taken first come first served: a request's rows continue where its last segment
    ended, and the next request starts only once the previous one's prompt is complete in this step.  A request's prompt is
    complete (its first token is due) in the step whose segment ends at its last row."""
    if budget < 1:
        raise ValueError(f"prefill_chunk must be >= 1, got {budget}")
    out = []
    for r, done, total in pending:
        if budget == 0:
            break
        n = min(total - done, budget)
        if n > 0:
            out.append((r, done, n))
            budget -= n
    return out


class PagePool:
    """pages [0, n_pages) and a page table of `rows` rows x pages_per_row entries (host copy; DecodeStream uploads it).
    Entries past a row's pages are 0, a valid page that the kernels never read (they stop at the row's length)."""

    def __init__(self, n_pages, rows, pages_per_row, page_rows=PAGE_ROWS):
        if n_pages < 1:
            raise ValueError(f"kv_pages must be >= 1, got {n_pages}")
        if page_rows < 16 or page_rows & (page_rows - 1):
            raise ValueError(f"page_rows must be a power of two >= 16, got {page_rows}")
        self.n_pages, self.page_rows, self.pages_per_row = int(n_pages), int(page_rows), int(pages_per_row)
        self.refs = [0] * self.n_pages
        self._free = list(range(self.n_pages - 1, -1, -1))    # a stack: the lowest free page is taken first
        self.table = np.zeros((int(rows), self.pages_per_row), dtype=np.int32)
        self.owned = [None] * int(rows)                         # row -> its pages, None while the row is free

    @property
    def free_pages(self):
        return len(self._free)

    def need(self, prompt_rows, max_new_tokens, k=1):
        """pages a request of k beams reserves: ceil((T + max_new_tokens) / P) for one beam; with k beams the T // P full prompt
        pages once and each beam's pages from the prompt's last page on"""
        full = pages_for(prompt_rows + max_new_tokens, self.page_rows)
        shared = prompt_rows // self.page_rows
        return shared + k * (full - shared)

    def check_reserve(self, rows, prompt_rows, max_new_tokens):
        """raise (RuntimeError) unless reserve() of the same arguments would succeed; changes nothing"""
        busy = [r for r in rows if self.owned[r] is not None]
        if busy:
            raise RuntimeError(f"page-table rows {busy} are in use")
        if pages_for(prompt_rows + max_new_tokens, self.page_rows) > self.pages_per_row:
            raise RuntimeError(f"{prompt_rows} + {max_new_tokens} rows exceed the {self.pages_per_row} pages of a page-table row")
        n = self.need(prompt_rows, max_new_tokens, len(rows))
        if n > self.free_pages:
            raise RuntimeError(f"not enough free KV pages: the request needs {n}, {self.free_pages} of {self.n_pages} are free")

    def reserve(self, rows, prompt_rows, max_new_tokens):
        """pages of one request whose beams own the page-table `rows` (one row for a greedy or sampled request) -> the number of
        full prompt pages the rows share (rows [0, shared * P) of the first row are those of every row)"""
        self.check_reserve(rows, prompt_rows, max_new_tokens)
        full = pages_for(prompt_rows + max_new_tokens, self.page_rows)
        shared = prompt_rows // self.page_rows if len(rows) > 1 else 0
        common = [self._free.pop() for _ in range(shared)]
        for r in rows:
            pages = common + [self._free.pop() for _ in range(full - shared)]
            for p in pages:
                self.refs[p] += 1
            self.owned[r] = pages
            self.table[r, :len(pages)] = pages
            self.table[r, len(pages):] = 0
        return shared

    def release(self, rows):
        """return the pages of page-table `rows` (a page shared by other rows stays until its last row is released)"""
        for r in rows:
            pages, self.owned[r] = self.owned[r], None
            for p in pages or ():
                self.refs[p] -= 1
                if self.refs[p] == 0:
                    self._free.append(p)
            self.table[r] = 0

    def release_all(self):
        self.release([r for r, o in enumerate(self.owned) if o is not None])

    def check(self):
        """assert the pool's invariants: every page is free xor referenced, and each reference count is the number of rows
        that list the page"""
        count = [0] * self.n_pages
        for pages in self.owned:
            for p in pages or ():
                count[p] += 1
        assert count == self.refs, "reference counts differ from the rows' pages"
        free = set(self._free)
        assert len(free) == len(self._free), "a page is free twice"
        assert all((c == 0) == (p in free) for p, c in enumerate(count)), "a page is both free and owned, or neither"


class GrowingPool(PagePool):
    """PagePool whose requests grow a page at a time and are swapped to a host area of `swap_pages` pages when the pool runs dry.

    Requests are named by a key (the stream's request id).  The pool tracks each running request's next write position (the
    same for all its beams: they grow in lockstep, so a fork's copy always finds its destination rows); schedule() is called
    once before each step and advances it.

    Admission rule: a request is admitted only while no request waits to resume, if its prompt pages plus the next step's
    growth of every running request (itself included) are free, and if the live requests but the smallest fit in the swap
    area at their full length (prompt plus max_new_tokens).  So a step never preempts the request it just admitted, and since
    the first running request is never a victim, the victims and the preempted requests always find room in the swap area, and
    that first request always finishes (every request's full length fits in the pool)."""

    def __init__(self, n_pages, rows, pages_per_row, swap_pages, page_rows=PAGE_ROWS):
        super().__init__(n_pages, rows, pages_per_row, page_rows)
        if swap_pages < 1:
            raise ValueError(f"kv_swap_pages must be >= 1, got {swap_pages}")
        self.swap_pages = int(swap_pages)
        self._swap_free = list(range(self.swap_pages - 1, -1, -1))
        self.running = []                                # keys in order of admission or resumption (newest last)
        self.preempted = []                              # keys in order of preemption (the next to resume first)
        self.rows_of, self.pos, self.full = {}, {}, {}   # key -> page-table rows / next write position / pages at full length
        self.swapped = {}                                # key of a preempted request -> each row's swap slots

    @property
    def free_swap_pages(self):
        return len(self._swap_free)

    def _growth(self, key, pos=None):
        """pages request `key`'s rows need before writing row pos (default its next write position)"""
        pos = self.pos[key] if pos is None else pos
        return sum(pos >= len(self.owned[r]) * self.page_rows for r in self.rows_of[key])

    def growth(self):
        """pages the next step's writes need"""
        return sum(self._growth(key) for key in self.running)

    def _refusal(self, rows, prompt_rows, max_new_tokens):
        if self.preempted:
            return f"{len(self.preempted)} preempted requests wait to resume"
        if any(self.owned[r] is not None for r in rows):
            return f"page-table rows {[r for r in rows if self.owned[r] is not None]} are in use"
        full = self.need(prompt_rows, max_new_tokens, len(rows))
        if pages_for(prompt_rows + max_new_tokens, self.page_rows) > self.pages_per_row or full > self.n_pages:
            return f"{prompt_rows} + {max_new_tokens} rows exceed the pool or a page-table row"
        grow = len(rows) if prompt_rows % self.page_rows == 0 else 0
        n = self.need(prompt_rows, 0, len(rows)) + grow + self.growth()
        if n > self.free_pages:
            return f"not enough free KV pages: the request and the next step need {n}, {self.free_pages} of {self.n_pages} are free"
        live = list(self.full.values()) + [full]
        if sum(live) - min(live) > self.swap_pages:
            return f"the swap area of {self.swap_pages} pages cannot hold the live requests but the smallest"
        return None

    def can_admit(self, rows, prompt_rows, max_new_tokens):
        return self._refusal(rows, prompt_rows, max_new_tokens) is None

    def check_admit(self, rows, prompt_rows, max_new_tokens):
        """raise (RuntimeError) unless admit() of the same arguments would succeed; changes nothing"""
        why = self._refusal(rows, prompt_rows, max_new_tokens)
        if why is not None:
            raise RuntimeError(why)

    def admit(self, key, rows, prompt_rows, max_new_tokens):
        """the pages prompt_rows fill for request `key` on page-table `rows` -> the number of full prompt pages the rows share"""
        self.check_admit(rows, prompt_rows, max_new_tokens)
        shared = self.reserve(rows, prompt_rows, 0)
        self.running.append(key)
        self.rows_of[key], self.pos[key] = list(rows), int(prompt_rows)
        self.full[key] = self.need(prompt_rows, max_new_tokens, len(rows))
        return shared

    def finish(self, key):
        """request `key` ended: its pages return to the pool"""
        self.release(self.rows_of.pop(key))
        self.running.remove(key)
        del self.pos[key], self.full[key]

    def _distinct(self, key):
        return list(dict.fromkeys(p for r in self.rows_of[key] for p in self.owned[r]))

    def swap_out(self, key):
        """preempt running request `key` -> [(page, swap slot)] to copy out; its pages are free once the copy ran"""
        pages = self._distinct(key)
        if len(pages) > self.free_swap_pages:
            raise RuntimeError(f"the swap area has {self.free_swap_pages} free pages, request {key} holds {len(pages)}")
        slot = {p: self._swap_free.pop() for p in pages}
        rows = self.rows_of.pop(key)
        self.swapped[key] = [[slot[p] for p in self.owned[r]] for r in rows]
        self.release(rows)
        self.running.remove(key)
        self.preempted.append(key)
        return [(p, slot[p]) for p in pages]

    def _resume_need(self, key):
        slots = len({s for row in self.swapped[key] for s in row})
        grow = sum(self.pos[key] >= len(row) * self.page_rows for row in self.swapped[key])
        return slots + grow

    def swap_in(self, key, rows):
        """resume preempted request `key` on page-table `rows` -> [(swap slot, page)] to copy in; the rows share the pages
        they shared before"""
        if key != (self.preempted[0] if self.preempted else None):
            raise RuntimeError(f"request {key} is not the next to resume")
        if len(rows) != len(self.swapped[key]) or any(self.owned[r] is not None for r in rows):
            raise RuntimeError(f"page-table rows {list(rows)} are not {len(self.swapped[key])} free rows")
        n = self._resume_need(key) + self.growth()
        if n > self.free_pages:
            raise RuntimeError(f"not enough free KV pages to resume request {key}: {n} needed, {self.free_pages} free")
        held = self.swapped.pop(key)
        page = {s: self._free.pop() for s in dict.fromkeys(s for row in held for s in row)}
        for r, row in zip(rows, held):
            pages = [page[s] for s in row]
            for p in pages:
                self.refs[p] += 1
            self.owned[r] = pages
            self.table[r, :len(pages)] = pages
            self.table[r, len(pages):] = 0
        self._swap_free.extend(reversed(list(page)))
        self.preempted.pop(0)
        self.running.append(key)
        self.rows_of[key] = list(rows)
        return list(page.items())

    def grow(self):
        """append a page to every running row whose next write starts a page it lacks -> whether the table changed"""
        rows = [r for key in self.running for r in self.rows_of[key] if self.pos[key] >= len(self.owned[r]) * self.page_rows]
        if len(rows) > self.free_pages:
            raise RuntimeError(f"the step needs {len(rows)} new pages, {self.free_pages} are free")
        for r in rows:
            if len(self.owned[r]) >= self.pages_per_row:
                raise RuntimeError(f"page-table row {r} is full")
        for r in rows:
            p = self._free.pop()
            self.refs[p] += 1
            self.table[r, len(self.owned[r])] = p
            self.owned[r].append(p)
        return bool(rows)

    def free_rows(self, k):
        """the first k free page-table rows, or None when fewer are free"""
        rows = [r for r, o in enumerate(self.owned) if o is None]
        return rows[:k] if len(rows) >= k else None

    def schedule(self):
        """the page work before one step, in order: resume preempted requests (oldest first, while their pages and the
        step's growth fit and free_rows finds their rows), else preempt the newest running requests until the growth fits,
        then grow.  Advances every running request's write position by the step's one row.
        -> (resumed [(key, rows, [(slot, page)])], preempted [(key, [(page, slot)])], table changed)"""
        resumed, preempted = [], []
        while self.preempted:
            key = self.preempted[0]
            rows = self.free_rows(len(self.swapped[key]))
            if rows is None or self._resume_need(key) + self.growth() > self.free_pages:
                break
            resumed.append((key, rows, self.swap_in(key, rows)))
        while self.growth() > self.free_pages:
            if len(self.running) < 2:
                raise RuntimeError("the pool cannot hold the oldest running request")
            assert not resumed, "a resumed request's growth was covered"
            key = self.running[-1]
            preempted.append((key, self.swap_out(key)))
        changed = self.grow() or bool(resumed)
        for key in self.running:
            self.pos[key] += 1
        return resumed, preempted, changed

    def release_all(self):
        super().release_all()
        self._swap_free = list(range(self.swap_pages - 1, -1, -1))
        self.running, self.preempted = [], []
        self.rows_of, self.pos, self.full, self.swapped = {}, {}, {}, {}

    def check(self):
        """PagePool.check, and: every swap slot is free xor held by one preempted request (its rows may share it), running
        requests own their rows, preempted ones none"""
        super().check()
        held = [s for key in self.swapped for s in dict.fromkeys(s for row in self.swapped[key] for s in row)]
        assert len(set(held)) == len(held), "a swap slot is held by two requests"
        assert sorted(held + self._swap_free) == list(range(self.swap_pages)), "a swap slot is both free and held, or neither"
        assert set(self.swapped) == set(self.preempted) and not set(self.running) & set(self.preempted)
        assert sorted(self.full) == sorted(self.running + self.preempted)
        rows = [r for key in self.running for r in self.rows_of[key]]
        assert len(set(rows)) == len(rows) and sorted(rows) == [r for r, o in enumerate(self.owned) if o is not None]
