"""Search-only V*Bench evaluation (vstar_b200.visual_search.main) against the REFERENCE's own `main`
(visual_search.py:520-564) run on the same synthetic tree with the same stub VSM (golden from tools/make_search_eval_golden.py).
The searches are independent, so every window of searches in flight must give the reference's per-target values."""
import json
import os

import pytest

from tests.helpers import FakeNLP, NumpyScorer
from tests.search_eval_helpers import ARGS, SPEC, SearchEvalRecordStub, SearchEvalStub, make_search_bench_folder
from vstar_b200 import noun_chunks

GOLD = os.path.join(os.path.dirname(__file__), "golden", "search_eval_golden.json")
N_TARGETS = sum(len(t) for items in SPEC.values() for *_, t in items)


@pytest.fixture(autouse=True)
def fake_nlp():
    noun_chunks.set_nlp(FakeNLP())           # the golden was made with the reference's spaCy pipeline replaced by FakeNLP
    yield
    noun_chunks.set_nlp(None)


@pytest.fixture(scope="module")
def gold():
    return json.load(open(GOLD))


def run(tmp_path, window, extra=(), vsm=None):
    from vstar_b200.visual_search import main
    folder = make_search_bench_folder(str(tmp_path / "bench"))
    traj = str(tmp_path / "traj.json")
    records = main(["--benchmark-folder", folder, "--searches-in-flight", str(window), "--search-batch", "8",
                    "--trajectory-json", traj, *extra] + ARGS, vsm=vsm or SearchEvalStub(), scorer=NumpyScorer())
    return records, json.load(open(traj))


def key(s):
    return (s["test_type"], s["image"], s["target_index"])


def check_samples(records, gold):
    assert len(records) == len(gold["samples"]) == N_TARGETS
    got = {key(r): r for r in records}
    for g in gold["samples"]:
        r = got[key(g)]
        assert (r["target"], r["gt_bbox"]) == (g["target"], g["gt_bbox"])
        assert (r["search_successful"], r["path_length"]) == (g["search_successful"], g["path_length"]), key(g)
        assert r["final_box"] == pytest.approx(g["final_box"], abs=1e-3), key(g)
        assert r["iou"] == pytest.approx(g["iou"], abs=1e-6), key(g)
        assert [e["bbox"] for e in r["expanded"]] == [e["bbox"] for e in g["expanded"]], key(g)
        assert [e["context_cue"] for e in r["expanded"]] == [e["context_cue"] for e in g["expanded"]], key(g)
        assert [e["score"] for e in r["expanded"]] == pytest.approx([e["score"] for e in g["expanded"]], abs=1e-6)


def test_golden_covers_every_outcome(gold):
    s = gold["samples"]
    per_image = {}
    for x in s:
        per_image[x["image"]] = per_image.get(x["image"], 0) + 1
    assert set(per_image.values()) == {1, 2, 3}
    assert any(x["search_successful"] and x["path_length"] == 1 and x["expanded"] == x["expanded"][:1] and x["iou"] > 0.5 for x in s)
    assert any(x["search_successful"] and x["path_length"] >= 4 for x in s)                  # deep search
    assert any(e["context_cue"] for x in s for e in x["expanded"])                           # weak-cue branch
    assert any(x["search_successful"] and len(x["expanded"]) > x["path_length"] for x in s)  # confidence_low fallback
    assert any(not x["search_successful"] for x in s)                                       # failed search
    assert any(x["iou"] > 0.5 for x in s) and any(x["search_successful"] and x["iou"] <= 0.5 for x in s)


@pytest.mark.parametrize("window", [1, 3, N_TARGETS])
def test_matches_reference_main(tmp_path, capsys, gold, window):
    records, traj = run(tmp_path, window)
    assert capsys.readouterr().out.splitlines() == gold["lines"]
    check_samples(records, gold)
    # the trajectory file holds the same records, in the reference's order (test type, then os.listdir order)
    assert traj["samples"] == json.loads(json.dumps(records))
    assert [r["test_type"] for r in records] == sorted(r["test_type"] for r in records)
    assert traj["searches_in_flight"] == window and traj["top1_acc"] == pytest.approx(float(gold["lines"][1].split(":")[1]))
    for r in records:
        assert r["latency_s"] >= 0 and r["evaluations"] >= len(r["expanded"])
        acc = 1.0 if r["search_successful"] and r["iou"] > 0.5 else 0
        assert r["accuracy"] == acc


def test_record_interface_matches_reference_main(tmp_path, capsys, gold):
    """the same run through the batched launch / finish record interface the CUDA VSM exposes"""
    records, _ = run(tmp_path, 4, vsm=SearchEvalRecordStub())
    assert capsys.readouterr().out.splitlines() == gold["lines"]
    check_samples(records, gold)


def test_visualization_files(tmp_path, gold):
    out = tmp_path / "vis"
    run(tmp_path, 3, extra=("--visualization", "--output_path", str(out)))
    files = sorted(os.path.relpath(os.path.join(d, f), out) for d, _, fs in os.walk(out) for f in fs)
    assert files == gold["visualization_files"]


def test_parse_args_defaults_are_the_reference():
    from vstar_b200.visual_search import parse_args
    a = parse_args([])
    # visual_search.py:28-52
    assert (a.version, a.benchmark_folder, a.visualization, a.output_path, a.confidence_low, a.confidence_high,
            a.target_cue_threshold, a.target_cue_threshold_decay, a.target_cue_threshold_minimum, a.minimum_size_scale,
            a.minimum_size, a.model_max_length, a.vision_tower, a.use_mm_start_end, a.conv_type) == (
        "craigwu/seal_vsm_7b", "vstar_bench", False, "", 0.3, 0.5, 6.0, 0.7, 3.0, 4.0, 224, 512, "openai/clip-vit-large-patch14",
        True, "llava_v1")
    assert a.trajectory_json is None and a.searches_in_flight >= 1


def test_missing_test_type_folder_raises(tmp_path):
    from vstar_b200.visual_search import main
    spec = {"direct_attributes": SPEC["direct_attributes"][:1]}
    folder = make_search_bench_folder(str(tmp_path / "bench"), spec)
    with pytest.raises(FileNotFoundError):
        main(["--benchmark-folder", folder] + ARGS, vsm=SearchEvalStub(), scorer=NumpyScorer())


def test_images_released_when_their_last_search_ends(tmp_path, monkeypatch):
    """each image is opened once, shared by its targets, and released as soon as its last search has ended"""
    events = []

    class Tracking(SearchEvalStub):
        def release(self, pil_img=None):
            events.append(("release", id(pil_img)))

    from vstar_b200 import visual_search as VS
    seen, keep = {}, []
    orig = VS.SearchState.__init__

    def init(self, image, *a, **k):
        keep.append(image)                   # no image is freed during the run, so no id is reused
        seen.setdefault(id(image), 0)
        seen[id(image)] += 1
        orig(self, image, *a, **k)

    monkeypatch.setattr(VS.SearchState, "__init__", init)
    run(tmp_path, 3, vsm=Tracking())
    n_images = sum(len(items) for items in SPEC.values())
    assert len(seen) == n_images and sorted(seen.values()) == sorted(len(t) for items in SPEC.values() for *_, t in items)
    assert sorted(i for _, i in events) == sorted(seen)


def test_module_cli_prints_the_reference_lines(tmp_path, capsys, gold, monkeypatch):
    """`python -m vstar_b200.visual_search ...` builds VSM(args) and prints the reference's two lines (VSM stubbed out: no checkpoint)"""
    import runpy
    import sys
    from vstar_b200 import vsm as vsm_mod
    folder = make_search_bench_folder(str(tmp_path / "bench"))
    built = []
    monkeypatch.setattr(vsm_mod, "VSM", lambda args: built.append(args.version) or SearchEvalRecordStub())
    monkeypatch.setattr(sys, "argv", ["visual_search", "--benchmark-folder", folder, "--version", "ckpt"] + ARGS)
    runpy.run_module("vstar_b200.visual_search", run_name="__main__")
    assert built == ["ckpt"]
    assert capsys.readouterr().out.splitlines() == gold["lines"]
