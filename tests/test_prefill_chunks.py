"""Chunked prefill of the paged decode stream, host side: kv_pages.plan_chunks' invariants on randomised queues and its edges,
DecodeStream's refusals of prefill_chunk (before any launch), and its plumbing through answer_open_many and the command line."""
import types

import numpy as np
import pytest

from tests import seal_open_helpers as H
from tests.helpers import StubVSM
from tests.test_seal_open import OpenStubLLM
from vstar_b200 import seal
from vstar_b200.kv_pages import plan_chunks


def run_queue(prompts, C, admit_at=None):
    """prefill the prompts (rows each; request i admitted before step admit_at[i]) with plan_chunks, checking every step ->
    {request: [(step, first row, rows)]}, {request: step its prompt completed}"""
    admit_at = admit_at or [0] * len(prompts)
    done = {i: 0 for i in range(len(prompts))}
    segs, complete = {i: [] for i in range(len(prompts))}, {}
    step = 0
    while len(complete) < len(prompts):
        pending = [(i, done[i], T) for i, T in enumerate(prompts) if admit_at[i] <= step and i not in complete]
        plan = plan_chunks(pending, C)
        assert sum(n for _, _, n in plan) <= C
        assert sum(n for _, _, n in plan) == min(C, sum(T - d for _, d, T in pending))   # the budget is used while rows wait
        order = [i for i, _, _ in pending]
        for k, (i, lo, n) in enumerate(plan):
            assert i == order[k]                            # first come first served: no request skipped ...
            assert n >= 1 and lo == done[i]                 # ... rows in order, continuing where the last segment ended
            if k < len(plan) - 1:
                assert lo + n == prompts[i]                 # ... and the next one starts only once this one is complete
            segs[i].append((step, lo, n))
            done[i] = lo + n
            if done[i] == prompts[i]:
                complete[i] = step
        step += 1
    return segs, complete


@pytest.mark.parametrize("seed", range(40))
def test_plan_chunks_invariants_on_random_queues(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 12))
    prompts = rng.integers(1, 900, n).tolist()
    C = int(rng.choice([1, 7, 64, 100, 256, 512, 2000]))
    admit_at = sorted(rng.integers(0, 30, n).tolist())
    segs, complete = run_queue(prompts, C, admit_at)
    for i, T in enumerate(prompts):
        rows = [r for _, lo, m in segs[i] for r in range(lo, lo + m)]
        assert rows == list(range(T))                       # every prompt row exactly once, in order
        assert complete[i] == segs[i][-1][0]                # the first token is due in the step of the last row, not before
        assert all(s >= admit_at[i] for s, _, _ in segs[i])
    for i in range(1, len(prompts)):                        # FCFS: a later request never completes before an earlier one
        assert complete[i] >= complete[i - 1]


@pytest.mark.parametrize("C", [1, 5, 64])
def test_plan_chunks_edges(C):
    # C = 1: one row per step; prompts of exactly C and C + 1 rows; C larger than every prompt
    segs, complete = run_queue([C, C + 1, 3], C)
    assert [m for _, _, m in segs[0]] == [C]
    assert [m for _, _, m in segs[1]] == [C, 1]
    assert complete[0] == 0 and complete[1] == 2
    segs, complete = run_queue([3, 2, 4], 1000)
    assert segs == {0: [(0, 0, 3)], 1: [(0, 0, 2)], 2: [(0, 0, 4)]} and complete == {0: 0, 1: 0, 2: 0}
    segs, _ = run_queue([4, 4], 1)
    assert segs[0] == [(s, s, 1) for s in range(4)] and segs[1] == [(4 + s, s, 1) for s in range(4)]
    assert plan_chunks([], 8) == []
    with pytest.raises(ValueError):
        plan_chunks([("a", 0, 5)], 0)


def test_prefill_chunk_refusals_before_any_launch():
    from vstar_b200 import _lib
    from vstar_b200.vqa import DecodeStream
    eng = types.SimpleNamespace(MAX_POSITIONS=2048)          # the refusals come before the engine is touched
    n0 = _lib.launches
    for kw in (dict(prefill_chunk=64), dict(prefill_chunk=64, kv_swap_pages=8)):
        with pytest.raises(ValueError, match="prefill_chunk|kv_swap_pages"):
            DecodeStream(eng, 4, 512, **kw)
    with pytest.raises(ValueError, match="kv_swap_pages"):
        DecodeStream(eng, 4, 512, kv_pages=16, kv_swap_pages=8, prefill_chunk=64)
    for bad in (0, -3, 2.5, True, "64"):
        with pytest.raises((ValueError, TypeError)):
            DecodeStream(eng, 4, 512, kv_pages=16, prefill_chunk=bad)
    assert _lib.launches == n0


class KwStubLLM(OpenStubLLM):
    """the scripted VQA LLM of test_seal_open, recording the stream keywords each decode phase receives"""

    def __init__(self):
        super().__init__()
        self.kw = []

    def _decode_stream(self, reqs, max_new_tokens, slots, **kw):
        self.kw.append(kw)
        yield from super()._decode_stream(reqs, max_new_tokens, slots)


def test_answer_open_many_passes_prefill_chunk_only_when_set(monkeypatch):
    from vstar_b200 import visual_search as VS
    monkeypatch.setattr(VS.SearchController, "stream", lambda self, states, window=None: ((st, H.fake_search(st.target, st.image))
                                                                                          for st in states))
    items = [(H.case_image(c), c[0]) for c in H.CASES]
    want = seal.answer_open_many(OpenStubLLM(), StubVSM(), items)          # the greedy-only signature still serves the default
    for kw in (dict(), dict(kv_pages=40), dict(kv_pages=40, prefill_chunk=256)):
        llm = KwStubLLM()
        got = seal.answer_open_many(llm, StubVSM(), items, **kw)
        assert llm.kw and all(k == kw for k in llm.kw), llm.kw
        assert [g[0] for g in got] == [w[0] for w in want] and [g[3] for g in got] == [w[3] for w in want]


def test_cli_prefill_chunk(monkeypatch, tmp_path):
    p = seal.build_parser()
    assert p.parse_args(["--image", "x.png", "--question", "q"]).prefill_chunk is None
    assert p.parse_args(["--image", "x.png", "--question", "q", "--kv-pages", "64", "--prefill-chunk", "256"]).prefill_chunk == 256
    seen = []

    def fake(vqa_llm, vsm, items, **kw):
        seen.append(kw)
        return [("a", None, None, None)] * len(items)
    monkeypatch.setattr(seal, "answer_open_many", fake)
    img = tmp_path / "x.png"
    from PIL import Image
    Image.new("RGB", (8, 8)).save(img)
    for extra, want in (([], None), (["--kv-pages", "64", "--prefill-chunk", "128"], 128)):
        seal.main(["--image", str(img), "--question", "q", "--output-path", str(tmp_path / "o.json"), *extra], vqa_llm=object(),
                  vsm=object())
        assert seen[-1]["prefill_chunk"] == want
