"""Page allocator of the paged decode stream (DecodeStream(kv_pages=N)), pure host code.

The pool holds N pages of PAGE_ROWS k|v rows per layer.  A decode row (a greedy or sampled request, or one beam of a beam
request) owns one row of the page table: the pages that hold its keys, in order, so key j sits in page table[row][j // P] at
row j % P.  Pages are reserved at admission for the whole request, prompt plus max_new_tokens, and never grow or move while it
runs; they return to the pool when it ends or the stream closes.

A beam request of k beams shares the full pages of its prompt among its beams (a reference count per page) and gives every beam
private pages from the prompt's last, partly filled page on: the beams write their generated rows there, and a fork copies the
parent's generated rows into the child's private pages, so no page a step writes is shared.
"""
from __future__ import annotations

import numpy as np

PAGE_ROWS = 64                                   # rows per page: a power of two >= 16 (the kernels' page_rows)


def pages_for(rows, page_rows=PAGE_ROWS):
    return -(-int(rows) // page_rows)


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
