"""Open-ended SEAL answering (vstar_b200.seal.answer_open / answer_open_many) against the reference demo's own inference()
(app.py:130-233): tests/golden/seal_open_golden.json is that function run on the six cases of tests/seal_open_helpers.py
(tools/make_seal_open_golden.py), with the same scripted model answers and search outcomes.  Pinned per case: the four
outputs (the annotated image byte for byte), every request handed to the VQA LLM (prompt ids, the image it is given, its
pixels and the object crops' pixels, images_long / objects_long, max_new_tokens, greedy decoding) and every search's
arguments.  Plus the command line's flags and its JSONL -> JSON round trip."""
import json
import os

import numpy as np
import pytest

from tests import seal_open_helpers as H
from tests.helpers import StubVSM
from vstar_b200 import seal
from vstar_b200.vqa import VQA_LLM, _clip_preprocess, _Proc

GOLD = os.path.join(os.path.dirname(__file__), "golden", "seal_open_golden.json")


class OpenStubLLM(VQA_LLM):
    """VQA_LLM with its prompt building, crops and answer post-processing, on the character tokenizer; the decode stream is
    replaced by the scripted model, which records every request and completes them in reverse order"""

    def __init__(self):
        self.tokenizer, self.image_processor, self.eos = H.CharTokenizer(), _Proc(), 2
        self.log = []

    def _decode_stream(self, reqs, max_new_tokens, slots):
        for i, (ids, image, crops, il, ol) in reversed(list(enumerate(reqs))):
            self.log.append(dict(ids=list(ids), image=H.image_sha(image), images=H.pixel_record(_clip_preprocess(image)),
                                 object_features=None if crops is None else H.pixel_record(crops), images_long=il,
                                 objects_long=ol, max_new_tokens=max_new_tokens))
            yield i, H.answer_ids(ids)


@pytest.fixture
def run(monkeypatch):
    from vstar_b200 import visual_search as VS
    searched = []

    def stream(self, states, window=None):
        for st in states:
            searched.append(dict(name=st.target, image=H.image_sha(st.image), smallest_size=st.smallest_size,
                                 confidence_low=st.confidence_low))
            yield st, H.fake_search(st.target, st.image)
    monkeypatch.setattr(VS.SearchController, "stream", stream)

    def go(**kw):
        llm = OpenStubLLM()
        items = [(H.case_image(c), c[0]) for c in H.CASES]
        return llm, seal.answer_open_many(llm, StubVSM(), items, **kw), searched
    return go


def same_pixels(got, want):
    assert got["shape"] == want["shape"]
    assert np.allclose(got["channel_sums"], want["channel_sums"], rtol=0, atol=1.0)
    assert np.allclose(got["samples"], want["samples"], rtol=0, atol=2.5e-3)      # one fp16 step at |x| <= 2.6


def test_answer_open_many_equals_the_reference_inference(run):
    gold = json.load(open(GOLD))["cases"]
    llm, outs, searched = run(slots=2, searches_in_flight=2)
    tok = H.CharTokenizer()
    calls = {}
    for rec in llm.log:
        text = tok.decode(rec["ids"])
        q = text.split("\n")[-1][:-len(" ASSISTANT:")]
        calls.setdefault(q, []).append(rec)
    assert len(llm.log) == sum(len(g["calls"]) for g in gold) == 11
    for g, out in zip(gold, outs):
        assert [out[0], out[1], H.array_sha(out[2]), out[3]] == g["outputs"], g["question"]
        mine = sorted(calls[g["question"]], key=lambda r: tok.decode(r["ids"]).count(H.FOCUS_MSG))      # direct, then final
        assert len(mine) == len(g["calls"])
        for got, want in zip(mine, g["calls"]):
            assert got["ids"] == want["ids"] and got["image"] == want["image"]
            assert got["images_long"] == want["images_long"] and got["objects_long"] == want["objects_long"]
            assert got["max_new_tokens"] == want["max_new_tokens"] == 512
            assert want["temperature"] == 0 and not want["do_sample"] and want["num_beams"] == 1      # greedy, as the stream decodes
            same_pixels(got["images"], want["images"])
            assert (got["object_features"] is None) == (want["object_features"] is None)
            if got["object_features"] is not None:
                same_pixels(got["object_features"], want["object_features"])
    want_searches = [dict(name=s["name"], image=s["image"], smallest_size=s["smallest_size"], confidence_low=s["confidence_low"])
                     for g in gold for s in g["searches"]]
    assert searched == want_searches
    assert all(s["target_bbox"] is None and s["other"] == [] for g in gold for s in g["searches"])


def test_answer_open_is_answer_open_many_of_one(run):
    _, outs, _ = run()
    for c, out in zip(H.CASES, outs):
        one = seal.answer_open(OpenStubLLM(), StubVSM(), H.case_image(c), c[0])
        assert one[0] == out[0] and one[1] == out[1] and one[3] == out[3]
        assert H.array_sha(one[2]) == H.array_sha(out[2])


def test_cli_flags_and_jsonl_round_trip(run, tmp_path):
    p = seal.build_parser()
    a = p.parse_args(["--image", "x.png", "--question", "what"])
    assert (a.vqa_model_path, a.vsm_model_path, a.conv_type, a.minimum_size_scale, a.minimum_size) == \
        ("craigwu/seal_vqa_7b", "craigwu/seal_vsm_7b", "v1", 4.0, 224)
    assert a.vqa_dtype == "bf16" and a.vqa_load_4bit is False
    with pytest.raises(SystemExit):
        p.parse_args(["--image", "x.png", "--questions", "q.jsonl"])
    _, outs, _ = run()
    cases = H.CASES[:3]
    lines = []
    for i, c in enumerate(cases):
        path = tmp_path / f"im{i}.png"
        H.case_image(c).save(path)
        lines.append(json.dumps({"image": str(path), "question": c[0]}))
    (tmp_path / "q.jsonl").write_text("\n".join(lines) + "\n")
    out = tmp_path / "answers.json"
    recs = seal.main(["--questions", str(tmp_path / "q.jsonl"), "--output-path", str(out), "--save-images", str(tmp_path / "vis")],
                     vqa_llm=OpenStubLLM(), vsm=StubVSM())
    assert json.load(open(out)) == recs and [r["question"] for r in recs] == [c[0] for c in cases]
    for r, o in zip(recs, outs):
        assert (r["direct_answer"], r["search_summary"], r["final_answer"]) == (o[0], o[1], o[3])
    assert recs[0]["annotated_image"] is None
    from PIL import Image
    assert np.array_equal(np.array(Image.open(recs[2]["annotated_image"])), outs[2][2])
