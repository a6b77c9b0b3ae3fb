"""The pipelined open-ended SEAL answering (vstar_b200.seal.answer_open_stream) on the CPU, with fakes of its two sessions:
(1) on the six scripted cases of tests/golden/seal_open_golden.json it equals the reference demo's own inference() in the
comparisons tests/test_seal_open.py makes for answer_open_many; (2) its schedule: a question's searches start after its
direct answer, its final answer after its last search, finals overlap other questions' work, questions are yielded as they
complete and the results equal answer_open_many's, also with no items, slots = 1 and failed searches; (3) the search
controller's step-wise session (SearchController.session): searches added late end as stream() ends them, and stream() over
the session launches the batches it launched before; (4) the command line's --pipeline."""
import json
import os

import numpy as np
import pytest
import torch

from tests import seal_open_helpers as H
from tests.helpers import FakeNLP, NumpyScorer, RecordStub, StubVSM, synth_image
from vstar_b200 import noun_chunks, seal
from vstar_b200 import visual_search as VS
from vstar_b200.beam import DEFAULT_EARLY_STOPPING, DEFAULT_LENGTH_PENALTY
from vstar_b200.vqa import DEFAULT_TOP_K, VQA_LLM, _clip_preprocess, _Proc, draw_seeds

GOLD = os.path.join(os.path.dirname(__file__), "golden", "seal_open_golden.json")
G = os.path.join(os.path.dirname(__file__), "golden")


def steps_for(text):
    """decode steps a scripted answer takes: spread, so that answers end out of admission order"""
    return 1 + sum(map(ord, text)) % 4


class PipeLLM(VQA_LLM):
    """VQA_LLM's prompt building, crops and answer post-processing on the character tokenizer.  Its decode paths are the
    scripted model: _decode_stream for answer_open_many (as in test_seal_open), and answer_session -> FakeAnswers for
    answer_open_stream.  Every request handed to either is logged with what the reference golden pins."""

    def __init__(self, events=None):
        self.tokenizer, self.image_processor, self.eos = H.CharTokenizer(), _Proc(), 2
        self.log, self.events, self.sessions = [], events if events is not None else [], []
        self.top_k, self.length_penalty, self.early_stopping = DEFAULT_TOP_K, DEFAULT_LENGTH_PENALTY, DEFAULT_EARLY_STOPPING

    def record(self, ids, image, crops, il, ol, max_new_tokens):
        self.log.append(dict(ids=list(ids), image=H.image_sha(image), images=H.pixel_record(_clip_preprocess(image)),
                             object_features=None if crops is None else H.pixel_record(crops), images_long=il, objects_long=ol,
                             max_new_tokens=max_new_tokens))

    def _decode_stream(self, reqs, max_new_tokens, slots):
        for i, (ids, image, crops, il, ol) in reversed(list(enumerate(reqs))):
            self.record(ids, image, crops, il, ol, max_new_tokens)
            yield i, H.answer_ids(ids)

    def answer_session(self, max_new_tokens, slots, max_positions=None, num_beams=1, **kw):
        s = FakeAnswers(self, max_new_tokens, slots, max_positions, num_beams, kw)
        self.sessions.append(s)
        return s


class FakeAnswers:
    """AnswerSession's surface on the scripted model: `slots` answers at a time, each ending after steps_for(its text) steps"""

    def __init__(self, llm, max_new_tokens, slots, max_positions, num_beams, kw):
        self.llm, self.max_new_tokens, self.slots = llm, max_new_tokens, slots
        self.max_positions, self.num_beams, self.kw = max_positions, num_beams, kw
        self.running, self.settings, self.closed = [], [], False
        self.refuse_if = None                     # question text -> refuse it

    def request(self, item):
        image, question, crops, il, ol = item
        return (self.llm._prompt_ids(question), image, crops, il, ol)

    def refuse(self, prompts, what):
        for ids, *_ in prompts:
            if self.refuse_if is not None and self.refuse_if(H.CharTokenizer().decode(ids)):
                raise ValueError(f"kv_pages = {self.kw.get('kv_pages')} cannot hold {what}")

    def fits(self, p):
        return len(self.running) < self.slots

    def admit(self, key, p, **settings):
        assert not self.closed and self.fits(p)
        ids, image, crops, il, ol = p
        self.llm.record(ids, image, crops, il, ol, self.max_new_tokens)
        self.llm.events.append(("admit", key))
        self.settings.append((key, settings))
        out = H.answer_ids(ids)
        self.running.append([key, out, steps_for(self.llm._answer_text(out))])

    @property
    def busy(self):
        return bool(self.running)

    def step(self):
        assert self.running
        done = []
        for r in self.running:
            r[2] -= 1
            if r[2] == 0:
                done.append((r[0], self.llm._answer_text(r[1])))
                self.llm.events.append(("end", r[0]))
        self.running = [r for r in self.running if r[2] > 0]
        return done

    def close(self):
        self.closed = True


class FakeSearches:
    """SearchSession's surface: `window` searches at a time, each ending after 1 + crc(name) % 3 steps with fake_search"""

    def __init__(self, window, events, searched):
        self.window, self.events, self.searched = window, events, searched
        self.queue, self.active = [], []

    def add(self, st):
        self.searched.append(dict(name=st.target, image=H.image_sha(st.image), smallest_size=st.smallest_size,
                                  confidence_low=st.confidence_low))
        self.events.append(("search", st.owner))
        self.queue.append(st)

    @property
    def idle(self):
        return not (self.queue or self.active)

    def step(self):
        while self.queue and len(self.active) < self.window:
            st = self.queue.pop(0)
            self.active.append([st, 1 + sum(map(ord, st.target)) % 3])
        done = []
        for a in self.active:
            a[1] -= 1
            if a[1] == 0:
                self.events.append(("found", a[0].owner))
                done.append((a[0], H.fake_search(a[0].target, a[0].image)))
        self.active = [a for a in self.active if a[1] > 0]
        return done


@pytest.fixture
def run(monkeypatch):
    """-> go(items=None, **kw) running answer_open_stream on the fakes: (llm, [(index, outputs)] in yield order, searches, events)"""
    def go(items=None, **kw):
        events, searched = [], []
        monkeypatch.setattr(VS.SearchController, "session", lambda self, window=None, feed=None: FakeSearches(window, events, searched))
        llm = PipeLLM(events)
        items = [(H.case_image(c), c[0]) for c in H.CASES] if items is None else items
        got = []
        for i, out in seal.answer_open_stream(llm, StubVSM(), items, **kw):
            events.append(("yield", i))
            got.append((i, out))
        return llm, got, searched, events
    return go


def phased(monkeypatch, items=None, **kw):
    monkeypatch.setattr(VS.SearchController, "stream", lambda self, states, window=None: ((st, H.fake_search(st.target, st.image))
                                                                                          for st in states))
    items = [(H.case_image(c), c[0]) for c in H.CASES] if items is None else items
    return seal.answer_open_many(PipeLLM(), StubVSM(), items, **kw)


def same_pixels(got, want):
    assert got["shape"] == want["shape"]
    assert np.allclose(got["channel_sums"], want["channel_sums"], rtol=0, atol=1.0)
    assert np.allclose(got["samples"], want["samples"], rtol=0, atol=2.5e-3)      # one fp16 step at |x| <= 2.6


def keyed(outs):
    """the four outputs per item, the annotated image by its bytes"""
    return [(o[0], o[1], H.array_sha(o[2]), o[3]) for o in outs]


def in_order(got, n):
    out = [None] * n
    for i, o in got:
        assert out[i] is None
        out[i] = o
    return out


def test_answer_open_stream_equals_the_reference_inference(run):
    gold = json.load(open(GOLD))["cases"]
    llm, got, searched, _ = run(slots=2, searches_in_flight=2)
    outs = in_order(got, len(gold))
    tok = H.CharTokenizer()
    calls = {}
    for rec in llm.log:
        q = tok.decode(rec["ids"]).split("\n")[-1][:-len(" ASSISTANT:")]
        calls.setdefault(q, []).append(rec)
    assert len(llm.log) == sum(len(g["calls"]) for g in gold) == 11
    for g, out in zip(gold, outs):
        assert [out[0], out[1], H.array_sha(out[2]), out[3]] == g["outputs"], g["question"]
        mine = calls[g["question"]]                    # admitted direct, then final
        assert [tok.decode(r["ids"]).count(H.FOCUS_MSG) for r in mine] == list(range(len(mine)))
        assert len(mine) == len(g["calls"])
        for rec, want in zip(mine, g["calls"]):
            assert rec["ids"] == want["ids"] and rec["image"] == want["image"]
            assert rec["images_long"] == want["images_long"] and rec["objects_long"] == want["objects_long"]
            assert rec["max_new_tokens"] == want["max_new_tokens"] == 512
            assert want["temperature"] == 0 and not want["do_sample"] and want["num_beams"] == 1
            same_pixels(rec["images"], want["images"])
            assert (rec["object_features"] is None) == (want["object_features"] is None)
            if rec["object_features"] is not None:
                same_pixels(rec["object_features"], want["object_features"])
    # searches start in the order direct answers end: compare each image's searches, in order
    want_searches = [dict(name=s["name"], image=s["image"], smallest_size=s["smallest_size"], confidence_low=s["confidence_low"])
                     for g in gold for s in g["searches"]]
    by_image = lambda recs: {im: [r for r in recs if r["image"] == im] for im in {r["image"] for r in recs}}      # noqa: E731
    assert by_image(searched) == by_image(want_searches) and len(searched) == len(want_searches)
    s, = llm.sessions
    assert s.closed and (s.slots, s.max_positions, s.num_beams) == (2, None, 1)
    assert s.kw == dict(kv_pages=None, kv_swap_pages=None, prefill_chunk=None) and all(st == {} for _, st in s.settings)


def test_schedule_stages_overlap_and_yield_order(run, monkeypatch):
    llm, got, searched, ev = run(slots=3, searches_in_flight=2)
    at = {e: t for t, e in enumerate(ev)}
    for i, c in enumerate(H.CASES):
        missing = list(c[5])
        if missing:
            for j in range(len(missing)):
                assert at[("end", (i, 0))] < at[("search", (i, j))]
            assert max(at[("found", (i, j))] for j in range(len(missing))) < at[("admit", (i, 1))] < at[("end", (i, 1))]
            assert at[("end", (i, 1))] < at[("yield", i)]
        else:
            assert ("admit", (i, 1)) not in at and at[("end", (i, 0))] < at[("yield", i)]
    # some final answer is admitted while another question's direct answer or search runs
    def running(k, t):
        spans = [(("admit", (k, 0)), ("end", (k, 0)))] + [(("search", (k, j)), ("found", (k, j))) for j in range(len(H.CASES[k][5]))]
        return any(at[a] < t < at[b] for a, b in spans)
    assert any(running(k, at[("admit", (i, 1))]) for i, c in enumerate(H.CASES) if c[5] for k in range(len(H.CASES)) if k != i)
    # yielded as each completes (in the step its last answer ends), not in input order
    for i, c in enumerate(H.CASES):
        t = at[("end", (i, 1 if c[5] else 0))]
        assert all(e[0] in ("end", "yield") for e in ev[t:at[("yield", i)]])
    order = [i for i, _ in got]
    assert sorted(order) == list(range(len(H.CASES))) and order != sorted(order)
    assert keyed(in_order(got, len(H.CASES))) == keyed(phased(monkeypatch, slots=3, searches_in_flight=2))


@pytest.mark.parametrize("kw", [dict(slots=1, searches_in_flight=1), dict(slots=16, searches_in_flight=8)])
def test_results_equal_answer_open_many(run, monkeypatch, kw):
    llm, got, _, ev = run(**kw)
    assert keyed(in_order(got, len(H.CASES))) == keyed(phased(monkeypatch, **kw))
    assert llm.sessions[0].slots == min(kw["slots"], len(H.CASES))
    if kw["slots"] == 1:                           # one answer at a time: every admission follows the previous answer's end
        adm = [t for t, e in enumerate(ev) if e[0] == "admit"]
        ends = [t for t, e in enumerate(ev) if e[0] == "end"]
        assert all(a > e for a, e in zip(adm[1:], ends))


def test_edge_cases(run, monkeypatch):
    llm, got, searched, _ = run(items=[])
    assert got == [] and llm.sessions == [] and searched == []
    # nothing missing: one direct answer, no search, no final
    llm, got, searched, ev = run(items=[(H.case_image(H.CASES[0]), H.CASES[0][0])])
    assert got == [(0, ("It is a cat.", None, None, None))] and searched == [] and len(llm.log) == 1
    # every search fails: the final prompt names the failures, as answer_open_many's does
    items = [(H.case_image(H.CASES[4]), H.CASES[4][0])]
    llm, got, searched, _ = run(items=items)
    want = phased(monkeypatch, items=items)[0]
    (i, out), = got
    assert i == 0 and keyed([out]) == keyed([want]) and out[1].endswith("Targets unable to locate after search: the key.")
    assert "not existent in the image" in H.CharTokenizer().decode(llm.log[-1]["ids"]) and len(searched) == 1


def test_refusal_names_the_question_and_closes_the_session(run, monkeypatch):
    events, searched = [], []
    monkeypatch.setattr(VS.SearchController, "session", lambda self, window=None, feed=None: FakeSearches(window, events, searched))
    llm = PipeLLM(events)
    orig = llm.answer_session

    def session(*a, **kw):
        s = orig(*a, **kw)
        s.refuse_if = lambda text: H.FOCUS_MSG in text and "Where is the dog" in text
        return s
    llm.answer_session = session
    items = [(H.case_image(c), c[0]) for c in H.CASES]
    with pytest.raises(ValueError, match=r"question 2 \('Where is the dog'\)"):
        list(seal.answer_open_stream(llm, StubVSM(), items, kv_pages=8))
    assert llm.sessions[0].closed and ("admit", (2, 1)) not in events


def test_sampling_seeds_and_beam_settings(run):
    torch.manual_seed(7)
    draws = draw_seeds(2 * len(H.CASES))
    torch.manual_seed(7)
    llm, got, _, _ = run(temperature=0.7, top_p=0.9)
    s = llm.sessions[0]
    assert len(s.settings) == 11
    for (i, stage), st in s.settings:
        assert st == dict(temperature=0.7, top_k=llm.top_k, top_p=0.9, seed=draws[2 * i + stage])
    llm, _, _, _ = run(num_beams=2, slots=4, kv_pages=40, kv_swap_pages=90)
    s = llm.sessions[0]
    assert s.num_beams == 2 and s.slots == 4 and s.kw == dict(kv_pages=40, kv_swap_pages=90, prefill_chunk=None)
    assert all(st == dict(num_beams=2, length_penalty=llm.length_penalty, early_stopping=llm.early_stopping) for _, st in s.settings)



# ---- the search controller's session ------------------------------------------------------------------------------------
TAGS = ["stub_3lvl", "stub_weakcue", "stub_mixcue", "edge_root_hit", "edge_deep_hit", "edge_tiny_unsure", "edge_wide", "edge_odd"]


@pytest.fixture
def fake_nlp():
    noun_chunks.set_nlp(FakeNLP())
    yield
    noun_chunks.set_nlp(None)


def golden_states():
    out = []
    for tag in TAGS:
        g = np.load(os.path.join(G, f"search_{tag}.npz"))
        st = VS.SearchState(synth_image(int(g["img_seed"]), int(g["w"]), int(g["h"])), "mug", int(g["smallest"]),
                            **json.loads(str(g["kw"])))
        st.tag = tag
        out.append(st)
    return out


def result_record(st, res):
    fs, pl, ok, av = res
    return (st.tag, [tuple(s["bbox"]) for s in st.search_path], list(fs["bbox"]), fs["detection_result"].tolist(), pl, ok,
            None if av is None else av.tolist(), [s.get("context_cue", "") for s in st.search_path])


def test_searches_added_late_end_as_in_stream(fake_nlp):
    want = {}
    for st, res in VS.SearchController(RecordStub(), NumpyScorer(), 8).stream(golden_states(), 3):
        want[st.tag] = result_record(st, res)
    ses = VS.SearchController(RecordStub(), NumpyScorer(), 8).session(3)
    later = golden_states()
    got, steps = {}, 0
    assert ses.idle
    while later or not ses.idle:
        if later and steps % 3 == 0:               # a new search every third step, while others run
            ses.add(later.pop(0))
        for st, res in ses.step():
            got[st.tag] = result_record(st, res)
        steps += 1
    assert got == want and ses.idle


def test_stream_over_the_session_launches_the_same_batches(fake_nlp):
    """batch sizes stream() launched on this input before it ran on the session (window 3, batch 8)"""
    ctl = VS.SearchController(RecordStub(), NumpyScorer(), 8)
    assert len(list(ctl.stream(iter(golden_states()), 3))) == len(TAGS)
    assert ctl.batches == [8] * 29 + [5] + [8] * 12 + [7, 6, 8, 5] + [8] * 5 + [5]
    one, two = [("vqa", 1), ("segmentation", 1)], [("vqa", 2), ("segmentation", 2)]
    assert ctl.cue_batches == one * 5 + two + one * 6


def test_stream_pulls_its_feed_only_when_there_is_room(fake_nlp):
    pulled = []

    def feed():
        for st in golden_states():
            pulled.append(st.tag)
            yield st
    seen = 0
    for st, _ in VS.SearchController(RecordStub(), NumpyScorer(), 8).stream(feed(), 2):
        seen += 1
        assert len(pulled) <= seen + 2
    assert seen == len(TAGS)


# ---- command line ----------------------------------------------------------------------------------------------------------
def test_cli_pipeline_flag(run, monkeypatch, tmp_path):
    p = seal.build_parser()
    assert p.parse_args(["--image", "x.png", "--question", "q"]).pipeline is False
    seen = []
    cases = H.CASES[:4]
    for k, c in enumerate(cases):
        H.case_image(c).save(tmp_path / f"im{k}.png")
    (tmp_path / "q.jsonl").write_text("".join(json.dumps({"image": str(tmp_path / f"im{k}.png"), "question": c[0]}) + "\n"
                                              for k, c in enumerate(cases)))
    flags = ["--kv-pages", "64", "--kv-swap-pages", "128", "--prefill-chunk", "256", "--temperature", "0.5", "--top_p", "0.8",
             "--num_beams", "3", "--slots", "5", "--searches-in-flight", "2", "--search-batch", "4"]
    want_kw = dict(slots=5, searches_in_flight=2, minimum_size_scale=4.0, minimum_size=224, search_batch=4, temperature=0.5, top_p=0.8,
                   num_beams=3, kv_pages=64, kv_swap_pages=128, prefill_chunk=256)
    outs = [(f"a{k}", None, None, None) if k % 2 else (f"b{k}", f"s{k}", np.full((3, 4, 3), k, np.uint8), f"f{k}") for k in range(4)]

    def fake_stream(vqa_llm, vsm, items, **kw):
        seen.append(("stream", kw))
        for k in (2, 0, 3, 1):
            yield k, outs[k]

    def fake_many(vqa_llm, vsm, items, **kw):
        seen.append(("many", kw))
        return outs
    monkeypatch.setattr(seal, "answer_open_stream", fake_stream)
    monkeypatch.setattr(seal, "answer_open_many", fake_many)
    recs = {}
    for extra in ([], ["--pipeline"]):
        out = tmp_path / f"o{len(extra)}.json"
        recs[len(extra)] = seal.main(["--questions", str(tmp_path / "q.jsonl"), "--output-path", str(out), *flags, *extra,
                                      "--save-images", str(tmp_path / f"vis{len(extra)}")], vqa_llm=object(), vsm=object())
        assert json.load(open(out)) == recs[len(extra)]
    assert seen == [("many", want_kw), ("stream", want_kw)]
    strip = lambda rs: [{k: v for k, v in r.items() if k != "annotated_image"} for r in rs]      # noqa: E731
    assert strip(recs[0]) == strip(recs[1]) and [bool(r["annotated_image"]) for r in recs[1]] == [True, False, True, False]
    assert list(recs[1][0]) == ["image", "question", "direct_answer", "search_summary", "final_answer", "annotated_image"]


def test_cli_pipeline_through_the_fakes(monkeypatch, tmp_path):
    """--pipeline on the real answer_open_stream writes the records the phased command line writes"""
    events, searched = [], []
    monkeypatch.setattr(VS.SearchController, "session", lambda self, window=None, feed=None: FakeSearches(window, events, searched))
    monkeypatch.setattr(VS.SearchController, "stream", lambda self, states, window=None: ((st, H.fake_search(st.target, st.image))
                                                                                          for st in states))
    for k, c in enumerate(H.CASES):
        H.case_image(c).save(tmp_path / f"im{k}.png")
    (tmp_path / "q.jsonl").write_text("".join(json.dumps({"image": str(tmp_path / f"im{k}.png"), "question": c[0]}) + "\n"
                                              for k, c in enumerate(H.CASES)))
    recs = [seal.main(["--questions", str(tmp_path / "q.jsonl"), "--output-path", str(tmp_path / f"o{k}.json"), *extra],
                      vqa_llm=PipeLLM(events), vsm=StubVSM()) for k, extra in enumerate(([], ["--pipeline"]))]
    assert recs[0] == recs[1] and len(recs[1]) == len(H.CASES)
