"""Differential tests of the host logic (integer geometry, priority queue order, prompt strings, placeholder splicing,
padding, patch geometry, noun chunks, visualisation files) against the reference modules (visual_search.py:226-283,
:378-389), on random inputs.  Every check is a driver that takes the functions under test and returns JSON-able results;
oracle/make_golden.py runs the drivers on the reference's own functions and stores their results (long lists as digests of
blocks of 500 items) in tests/golden/host_logic_reference.json, and the tests run the same drivers on ours and compare."""
import hashlib
import json
import os
import queue
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT) if ROOT not in sys.path else None

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "host_logic_reference.json")


def jsonable(x):
    return json.loads(json.dumps(x, default=lambda o: o.tolist() if hasattr(o, "tolist") else str(o)))


def digest(b):
    return hashlib.sha256(b).hexdigest()[:24]


def blockwise(x, n=500):
    """what the golden file stores: lists longer than n as one digest per n consecutive items, dicts key by key"""
    if isinstance(x, dict):
        return {k: blockwise(v, n) for k, v in x.items()}
    if isinstance(x, list) and len(x) > n:
        return [digest(json.dumps(x[i:i + n]).encode()) for i in range(0, len(x), n)]
    return x


def boxes(n, seed):
    rng = np.random.default_rng(seed)
    for _ in range(n):
        w, h = int(rng.integers(1, 9000)), int(rng.integers(1, 9000))
        yield [int(rng.integers(0, 5000)), int(rng.integers(0, 5000)), w, h]


SPLIT_BOXES = list(boxes(3000, 1)) + [[0, 0, 100, 200], [0, 0, 200, 100], [3, 5, 7, 14], [3, 5, 14, 7], [0, 0, 1, 1], [0, 0, 2, 3]]
QUESTIONS = ["Please locate the red mug in this image.", "According to the common sense knowledge and possible visual cues, what is "
             "the most likely location of the dog in the image?", "x"]


# ---------------------------------------------------------------- drivers (run on the reference by make_golden, on ours here)
def run_split_and_sub_patches(split_4subpatches, get_sub_patches):
    out = []
    for b in SPLIT_BOXES:
        nw, nh = split_4subpatches(b)
        got = get_sub_patches(b, nw, nh)
        out.append([[nw, nh], [list(got[0])] + list(got[1:])])
    return jsonable(out)


def run_refine_bbox_and_iou(refine_bbox, iou):
    rng = np.random.default_rng(2)
    out = []
    for _ in range(2000):
        W, H = int(rng.integers(10, 4000)), int(rng.integers(10, 4000))
        b = [float(rng.uniform(-50, W)), float(rng.uniform(-50, H)), float(rng.uniform(1, W)), float(rng.uniform(1, H))]
        c = [float(rng.uniform(0, W)), float(rng.uniform(0, H)), float(rng.uniform(1, W)), float(rng.uniform(1, H))]
        out.append([refine_bbox(list(b), W, H), iou(b, c)])
    return jsonable(out)


def run_prioritize_pop_order(Prioritize):
    """the expansion order IS the heap order of (Prioritize(-score, item)) incl. its tie behaviour (no tiebreak key)"""
    rng = np.random.default_rng(3)
    out = []
    for trial in range(50):
        scores = np.round(rng.uniform(0, 1, 40), 1 if trial % 2 else 3).astype(np.float32)      # many exact ties
        q, order = queue.PriorityQueue(), []
        for i, s in enumerate(scores):
            q.put(Prioritize(-s, i))
            if i % 3 == 2:                    # interleave pops with pushes like the search does
                order.append(q.get().item)
        while not q.empty():
            order.append(q.get().item)
        out.append(order)
    return out


def run_padding_and_patch_geometry(expand2square_vsm, expand2square_center, get_patch):
    """both expand2square variants (top-left paste for the VSM, centred for the VQA LLM) and VQA_LLM.get_patch"""
    from tests.helpers import synth_image
    out = dict(vsm=[], center=[], patch=[])
    for i, (w, h) in enumerate([(300, 200), (200, 300), (256, 256), (1, 9), (513, 512)]):
        img = synth_image(50 + i, w, h)
        bg = (122, 116, 104)
        out["vsm"].append(digest(np.ascontiguousarray(np.asarray(expand2square_vsm(img, bg))).tobytes()))
        a, la, ta = expand2square_center(img, bg)
        out["center"].append([la, ta, digest(np.ascontiguousarray(np.asarray(a)).tobytes())])
    rng = np.random.default_rng(5)
    for _ in range(2000):
        W, H = int(rng.integers(50, 3000)), int(rng.integers(50, 3000))
        bbox = [float(rng.uniform(0, W)), float(rng.uniform(0, H)), float(rng.uniform(1, W)), float(rng.uniform(1, H))]
        out["patch"].append([get_patch(None, bbox, W, H, patch_scale=scale) for scale in (None, 1.2, 0.5)])
    return jsonable(out)


def noun_chunk_phrases():
    from tests.helpers import VQA_ANSWERS, FakeNLP
    rng = np.random.default_rng(7)
    words = sorted(FakeNLP.NOUNS | FakeNLP.PRONS | FakeNLP.ADJS | FakeNLP.DETS | FakeNLP.PREPS | FakeNLP.RELS) + ["and", "somewhere", "high", "is"]
    phrases = [a.split("most likely to appear")[-1].strip().rstrip(".") for a in VQA_ANSWERS]
    for _ in range(3000):
        phrases.append(" ".join(rng.choice(words, size=int(rng.integers(1, 12)))))
    return phrases


def run_noun_chunks(extract_noun_chunks, get_noun_chunks, tranverse, filter_chunk_list, nlp):
    """extract_noun_chunks / get_noun_chunks / filter_chunk_list (visual_search.py:54-112) with the SAME deterministic parser
    on both sides (spaCy is not installed offline): random phrases from the rule parser's lexicon + hand-made trees.  The
    per-token results are stored as one digest per phrase."""
    out = dict(chunks=[], tokens=[], filtered=[])
    for ph in noun_chunk_phrases():
        out["chunks"].append(jsonable(extract_noun_chunks(ph)))
        per_tok = [[jsonable(get_noun_chunks(t)), jsonable(tranverse(t))] for t in nlp(ph)]
        out["tokens"].append(digest(json.dumps(per_tok).encode()))
    rng = np.random.default_rng(7)
    for _ in range(2000):
        chunks = [tuple(sorted(rng.integers(0, 30, 2).tolist())) for _ in range(int(rng.integers(0, 8)))]
        out["filtered"].append(jsonable(filter_chunk_list(chunks)))
    return out


def run_visualisation_files(visual_search):
    """visualize=True: the files visualize_search_path writes (visual_search.py:339-376) on the same stub search: file names,
    digests of the JPEG bytes and of context_cue.txt, path length and success flag"""
    from tests.helpers import StubVSM, synth_image
    out = []
    for seed, w, h, smallest, hot, kw in ((29, 640, 480, 224, None, dict(confidence_high=2.0, target_cue_threshold=9.5, target_cue_threshold_minimum=9.5)),
                                          (25, 700, 600, 224, "small", dict())):
        img = synth_image(seed, w, h)
        with tempfile.TemporaryDirectory() as d:
            r = visual_search(StubVSM(hot), img, "mug", [30, 40, 50, 60], smallest, visualize=True, save_path=d, **kw)
            files = sorted(os.listdir(d))
            out.append(dict(path_length=jsonable(r[1]), success=jsonable(r[2]), files=files,
                            digests=[digest(open(os.path.join(d, f), "rb").read()) for f in files]))
    return out


# ---------------------------------------------------------------- checks: our functions against the stored reference results
@pytest.fixture(scope="module")
def gold():
    return json.load(open(GOLD))


def check_split_and_sub_patches(gold):
    from vstar_b200 import visual_search as VS
    got = run_split_and_sub_patches(VS.split_4subpatches, VS.get_sub_patches)
    assert blockwise(got) == gold["split_and_sub_patches"]
    for b, ((nw, nh), (patches, *_)) in zip(SPLIT_BOXES, got):
        assert sum(p[2] * p[3] for p in patches) == b[2] * b[3]     # children tile the parent (the last one takes the remainder)
    shapes = [tuple(s) for s, _ in got]
    assert shapes.count((1, 4)) > 100 and shapes.count((4, 1)) > 100


def check_refine_bbox_and_iou(gold):
    from vstar_b200 import visual_search as VS
    assert blockwise(run_refine_bbox_and_iou(VS.refine_bbox, VS.iou)) == gold["refine_bbox_and_iou"]


def check_prioritize_pop_order_with_ties(gold):
    from vstar_b200 import visual_search as VS
    assert blockwise(run_prioritize_pop_order(VS.Prioritize)) == gold["prioritize_pop_order"]


def check_prompts_and_token_splicing(gold):
    """prompt strings of both conversation templates and the <image>/<object> placeholder splicing (they define T and the
    255-row offset): ours vs the reference's conversation.py / mm_utils.py, with the synthetic word-hash tokenizer on both"""
    from vstar_b200 import vqa, vsm
    from vstar_b200.config import tiny_config
    tok = vsm.SyntheticTokenizer(tiny_config())
    want = gold["prompts_and_token_splicing"]
    for i, q in enumerate(QUESTIONS):
        w = want[i]
        p = vsm.build_prompt(q, "llava_v1", True)
        assert p == w["vsm_v1"]
        assert [vsm.build_prompt(q, "llava_llama_2", use_se) for use_se in (True, False)] == w["vsm_llama_2"]
        ids = vsm.tokenizer_image_token(p, tok)
        assert ids == w["vsm_ids"] and ids.count(-200) == 1
        for j, answer in enumerate((None, "the mug is red")):
            qs = "<image>" + "\n" + "Additional visual information to focus on: mug <object> at location [0.1,0.2,0.3,0.4]; dog <object>.\n" + q
            pv = vqa.build_prompt_v1(qs, answer)
            assert pv == w["vqa"][j][0]
            ids = vqa.tokenizer_image_object_token(pv, tok)
            assert ids == w["vqa"][j][1] and ids.count(-200) == 1 and ids.count(-300) == 2


def check_padding_and_patch_geometry(gold):
    from vstar_b200 import seal, vqa, vsm
    got = run_padding_and_patch_geometry(vsm.expand2square, seal.expand2square_center, vqa.VQA_LLM.get_patch)
    assert blockwise(got) == gold["padding_and_patch_geometry"]


def check_noun_chunks(gold):
    from tests.helpers import FakeNLP
    from vstar_b200 import noun_chunks as NC
    nlp = FakeNLP()
    got = run_noun_chunks(lambda ph: NC.extract_noun_chunks(ph, nlp), NC.get_noun_chunks, NC.subtree_span, NC.filter_chunk_list, nlp)
    want = gold["noun_chunks"]
    for key in ("chunks", "tokens", "filtered"):
        assert blockwise(got[key]) == want[key], key
    n = [len(c) for c in got["chunks"]]
    assert sum(k > 1 for k in n) > 100 and sum(k == 1 for k in n) > 100 and sum(k == 0 for k in n) > 10


def check_visualisation_files(gold):
    from tests.helpers import FakeNLP, NumpyScorer
    from vstar_b200 import noun_chunks
    from vstar_b200 import visual_search as VS
    noun_chunks.set_nlp(FakeNLP())
    got = run_visualisation_files(lambda *a, **k: VS.visual_search(*a, scorer=NumpyScorer(), **k))
    assert blockwise(got) == gold["visualisation_files"]
    for case in got:
        f = case["files"]
        assert "whole_image.jpg" in f and "context_cue.txt" in f and any(x.endswith("_heatmap.jpg") for x in f), f


CHECKS = ["check_visualisation_files", "check_noun_chunks", "check_split_and_sub_patches", "check_refine_bbox_and_iou",
          "check_prioritize_pop_order_with_ties", "check_prompts_and_token_splicing", "check_padding_and_patch_geometry"]


@pytest.mark.parametrize("name", CHECKS)
def test_against_live_reference(gold, name):
    globals()[name](gold)
