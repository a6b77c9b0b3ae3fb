"""Host side of sampled and beam requests on the decode stream, without a GPU:
(1) beam.fork_slots, the copy-on-fork slot management beam_search and DecodeStream share, on hand-built beam transitions;
(2) seal's --temperature / --top_p / --num_beams flags and their way through answer_open_many to free_form_inference_stream and
    the decode stream; the greedy defaults keep the calls the greedy-only signatures accept;
(3) DecodeStream.admit's refusals, which raise before anything reaches the device."""
import pytest
import torch

from tests import seal_open_helpers as H
from tests.helpers import StubVSM
from vstar_b200 import _lib, seal
from vstar_b200.beam import fork_slots
from vstar_b200.vqa import DecodeStream, VQA_LLM, VQAEngine, _Proc


# ------------------------------------------------------------------------------------------------ fork_slots
def test_fork_slots_keeps_parents_and_claims_dead_beams():
    owned = [4, 9, 2, 7]
    old = [4, 9, 2, 7]                           # beam b on slot old[b]
    # beam 1 has three children, beam 3 one; beams 0 and 2 die
    new, forks = fork_slots(old, [(-1.0, 11, 1), (-1.1, 12, 3), (-1.2, 13, 1), (-1.3, 14, 1)], owned)
    assert new == [9, 7, 4, 2]                   # first children keep their parent's slot, later ones take dead slots in order
    assert forks == [(9, 4), (9, 2)]
    srcs, dsts = {s for s, _ in forks}, {d for _, d in forks}
    assert not srcs & dsts and len(dsts) == len(forks)


def test_fork_slots_without_forks_and_from_one_beam():
    # every beam survives with one child each, reordered: nothing is copied
    new, forks = fork_slots([3, 5, 8], [(0.0, 1, 2), (0.0, 2, 0), (0.0, 3, 1)], [3, 5, 8])
    assert new == [8, 3, 5] and forks == []
    # the first selection (one running beam on the prefilled slot): the other beams take the request's other slots; their
    # prompt rows are already there, so these forks copy no generated rows
    new, forks = fork_slots([6], [(0.0, 1, 0), (0.0, 2, 0), (0.0, 3, 0)], [6, 0, 1])
    assert new == [6, 0, 1] and forks == [(6, 0), (6, 1)]


def test_fork_slots_of_several_requests_never_read_a_written_slot():
    g = torch.Generator().manual_seed(0)
    for _ in range(200):
        k = int(torch.randint(2, 9, (1,), generator=g))
        owned = torch.randperm(32, generator=g)[:k].tolist()
        old = torch.randperm(k, generator=g).tolist()
        old = [owned[i] for i in old]
        parents = torch.randint(0, k, (k,), generator=g).tolist()
        new, forks = fork_slots(old, [(0.0, t, p) for t, p in enumerate(parents)], owned)
        assert sorted(new) == sorted(owned)      # the request keeps exactly its slots
        assert not {s for s, _ in forks} & {d for _, d in forks}
        for b, (s, p) in enumerate(zip(new, parents)):
            assert s == old[p] or (old[p], s) in forks


# ------------------------------------------------------------------------------------------------ seal flags
class RecordingLLM(VQA_LLM):
    """VQA_LLM on the character tokenizer whose decode stream is scripted; records the calls it receives"""

    def __init__(self):
        self.tokenizer, self.image_processor, self.eos = H.CharTokenizer(), _Proc(), 2
        self.top_k, self.length_penalty, self.early_stopping = 50, 1.0, False
        self.stream_calls, self.decode_calls = [], []

    def free_form_inference_stream(self, items, *args, **kw):
        self.stream_calls.append((len(items), args, kw))
        return super().free_form_inference_stream(items, *args, **kw)

    def _decode_stream(self, reqs, *args, **kw):
        self.decode_calls.append((len(reqs), args, kw))
        for i, (ids, *_rest) in enumerate(reqs):
            yield i, H.answer_ids(ids)


@pytest.fixture
def run(monkeypatch):
    from vstar_b200 import visual_search as VS

    def stream(self, states, window=None):
        for st in states:
            yield st, H.fake_search(st.target, st.image)
    monkeypatch.setattr(VS.SearchController, "stream", stream)

    def go(**kw):
        llm = RecordingLLM()
        items = [(H.case_image(c), c[0]) for c in H.CASES]
        return llm, seal.answer_open_many(llm, StubVSM(), items, slots=4, **kw)
    return go


def test_default_settings_keep_the_greedy_calls(run):
    llm, outs = run()
    assert len(llm.stream_calls) == 2            # direct answers, then final answers
    for n, args, kw in llm.stream_calls:
        assert args == () and kw == dict(max_new_tokens=seal.OPEN_MAX_NEW_TOKENS, slots=4)
    for n, args, kw in llm.decode_calls:
        assert args == (seal.OPEN_MAX_NEW_TOKENS, 4) and kw == {}
    spelled, _ = run(temperature=0, top_p=None, num_beams=1)     # the defaults spelled out are the defaults
    assert spelled.stream_calls == llm.stream_calls and spelled.decode_calls == llm.decode_calls


def test_sampling_settings_reach_both_phases(run):
    torch.manual_seed(5)
    llm, _ = run(temperature=0.7, top_p=0.9)
    assert len(llm.stream_calls) == 2
    for n, args, kw in llm.stream_calls:
        assert kw == dict(max_new_tokens=seal.OPEN_MAX_NEW_TOKENS, slots=4, temperature=0.7, top_p=0.9)
    seeds = []
    for n, args, kw in llm.decode_calls:
        st = kw["settings"]
        assert len(st) == n and all(s["temperature"] == 0.7 and s["top_p"] == 0.9 and s["top_k"] == 50 for s in st)
        seeds += [s["seed"] for s in st]
    torch.manual_seed(5)                         # one draw per item, in item order, before the first admission
    n0 = llm.decode_calls[0][0]
    assert seeds[:n0] == torch.empty(n0, dtype=torch.int64).random_().tolist()


def test_beam_settings_reach_both_phases(run):
    llm, _ = run(num_beams=3)
    assert [kw.get("num_beams") for _, _, kw in llm.stream_calls] == [3, 3]
    for n, args, kw in llm.decode_calls:
        assert kw["settings"] == [dict(num_beams=3, length_penalty=1.0, early_stopping=False)] * n


def test_stream_settings_refusals():
    llm = RecordingLLM()
    items = [(H.case_image(H.CASES[0]), "q", None, None, None)]
    with pytest.raises(NotImplementedError):
        list(llm.free_form_inference_stream(items, temperature=0.7, num_beams=2))
    with pytest.raises(ValueError):
        list(llm.free_form_inference_stream(items, num_beams=17))
    with pytest.raises(ValueError):
        list(llm.free_form_inference_stream(items, temperature=0.7, top_p=1.5))


def test_cli_flags_default_and_forward(monkeypatch, tmp_path):
    p = seal.build_parser()
    a = p.parse_args(["--image", "x.png", "--question", "what"])
    assert (a.temperature, a.top_p, a.num_beams) == (0, None, 1)
    a = p.parse_args(["--image", "x.png", "--question", "what", "--temperature", "0.7", "--top_p", "0.9", "--num_beams", "2"])
    assert (a.temperature, a.top_p, a.num_beams) == (0.7, 0.9, 2)
    got = {}

    def fake_many(vqa_llm, vsm, items, **kw):
        got.update(kw)
        return [("a", None, None, None) for _ in items]
    monkeypatch.setattr(seal, "answer_open_many", fake_many)
    path = tmp_path / "im.png"
    H.case_image(H.CASES[0]).save(path)
    seal.main(["--image", str(path), "--question", "what", "--output-path", str(tmp_path / "o.json"), "--temperature", "0.5",
               "--top_p", "0.8", "--num_beams", "1"], vqa_llm=RecordingLLM(), vsm=StubVSM())
    assert (got["temperature"], got["top_p"], got["num_beams"]) == (0.5, 0.8, 1)
    seal.main(["--image", str(path), "--question", "what", "--output-path", str(tmp_path / "o.json")], vqa_llm=RecordingLLM(),
              vsm=StubVSM())
    assert (got["temperature"], got["top_p"], got["num_beams"]) == (0, None, 1)


# ------------------------------------------------------------------------------------------------ admission refusals
class HostEngine:
    """the part of VQAEngine that DecodeStream.admit consults before it launches anything"""
    MAX_POSITIONS = 2048
    _beam_args = VQAEngine._beam_args

    def spliced_length(self, ids, n_crops=0, images_long=None, objects_long=None):
        return len(ids)


def host_stream(max_slots=3, busy=1, max_positions=100):
    st = DecodeStream.__new__(DecodeStream)
    st.engine, st.eos = HostEngine(), 2
    st.max_slots, st.max_positions = max_slots, max_positions
    st._cache = object()                         # open; admit must raise before it is touched
    st._slots = [object()] * busy + [None] * (max_slots - busy)
    return st


@pytest.mark.parametrize("kw,exc", [
    (dict(num_beams=2, temperature=0.7), NotImplementedError),
    (dict(num_beams=2, stop_ids=[5]), ValueError),
    (dict(num_beams=0), ValueError), (dict(num_beams=17), ValueError), (dict(num_beams=True), ValueError),
    (dict(num_beams=4), ValueError),                                       # more beams than the stream's slots
    (dict(num_beams=3), RuntimeError),                                     # 2 of 3 slots free
    (dict(num_beams=2, early_stopping="sometimes"), ValueError),
    (dict(temperature=0.7, top_k=-1), ValueError), (dict(temperature=0.7, top_p=1.5), ValueError),
])
def test_admit_refusals_raise_before_any_launch(kw, exc):
    st = host_stream()
    n0 = _lib.launches
    with pytest.raises(exc) as e:
        st.admit(([1, -200, 5], None, None, None, None), 4, **kw)
    if exc is RuntimeError:
        assert "no free slot" in str(e.value)
    with pytest.raises(_lib.VsbError, match="exceeds"):
        st.admit(([1] * 90, None, None, None, None), 11, num_beams=2)
    assert _lib.launches == n0
