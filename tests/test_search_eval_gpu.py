"""Search-only V*Bench evaluation on the CUDA VSM (tiny golden config): with W searches in flight, every target's result
equals that target's search run alone through visual_search().  This rests on the batch invariance of crop records
(tests/test_search_gpu.py::test_crop_records_do_not_depend_on_the_batch): a crop's record is the same whichever searches share
its batch.  The run also leaves no search image resident and gives its device memory back."""
import json
import os

import pytest
import torch

from tests.helpers import FakeNLP
from tests.search_eval_helpers import SPEC, make_search_bench_folder

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
N_TARGETS = sum(len(t) for items in SPEC.values() for *_, t in items)
# never confident (every search walks its whole tree, 1 or 21 nodes, then takes the confidence_low path); the root takes the
# weak-cue branch, deeper nodes the strong-cue one
THRESHOLDS = dict(confidence_high=2.0, target_cue_threshold=1e9, target_cue_threshold_decay=0.0, target_cue_threshold_minimum=-1e9)
ARGS = ["--minimum_size", "320", "--confidence_high", "2.0", "--target_cue_threshold", "1e9", "--target_cue_threshold_decay", "0.0",
        "--target_cue_threshold_minimum=-1e9"]
# device memory a finished evaluation may keep: nothing per search or per image; allocator rounding only
MEMORY_SLACK = 8 << 20


@pytest.fixture(scope="module", autouse=True)
def fake_nlp():
    from vstar_b200 import noun_chunks
    noun_chunks.set_nlp(FakeNLP())
    yield
    noun_chunks.set_nlp(None)


@pytest.fixture(scope="module")
def tiny_vsm():
    from oracle import vsm_oracle as O
    from vstar_b200.engine import VSMEngine, VSMWeights
    from vstar_b200.vsm import VSM
    j = json.load(open(os.path.join(G, "tiny_config.json")))
    cfg = O.VSMConfig(**j["cfg"])
    sd = O.synthetic_state_dict(cfg, seed=j["weight_seed"])
    eng = VSMEngine(VSMWeights.from_state_dict(cfg, sd))
    # eager engine calls only: a CUDA graph is captured on the third call of a batch shape and keeps its memory pool, which would
    # count as memory the evaluation kept (graph replays are bit-identical to eager calls: test_cuda_graph_replay_equals_eager)
    eng.graph_max_batch = 0
    prompt, ans = O.synthetic_prompt(cfg, n_text=24, seed=5)

    class GoldenVSM(VSM):
        def _ids(self, question):
            return prompt[0].tolist()

    return GoldenVSM(engine=eng, forced_answer_ids=ans.tolist(), frontier_batch=4)


@pytest.fixture(scope="module")
def folder(tmp_path_factory):
    return make_search_bench_folder(str(tmp_path_factory.mktemp("search_eval") / "bench"))


@pytest.fixture(scope="module")
def alone(tiny_vsm, folder):
    """every target searched on its own, one visual_search() call at a time (the reference's schedule)"""
    from PIL import Image
    from vstar_b200.seal import smallest_size_for
    from vstar_b200.visual_search import visual_search
    out = {}
    for test_type, items in SPEC.items():
        for name, *_, targets in items:
            img = Image.open(os.path.join(folder, test_type, name + ".png")).convert("RGB")
            smallest = smallest_size_for(img, 4.0, 320)
            for i, (gt, obj) in enumerate(targets):
                fs, pl, ok, _, st = visual_search(tiny_vsm, img, obj, gt, smallest, return_state=True, **THRESHOLDS)
                box = fs["detection_result"].clone()
                box[0] += fs["bbox"][0]
                box[1] += fs["bbox"][1]
                out[(test_type, name + ".png", i)] = dict(
                    search_successful=bool(ok), path_length=int(pl), final_box=[float(v) for v in box],
                    expanded=[dict(bbox=[int(v) for v in s["bbox"]], score=None if s["score"] is None else float(s["score"]),
                                   context_cue=s.get("context_cue")) for s in st.search_path])
            tiny_vsm.release(img)
    return out


@pytest.mark.parametrize("window", [1, 4, N_TARGETS])
def test_each_target_equals_its_search_alone(tiny_vsm, folder, alone, tmp_path, window):
    from vstar_b200.visual_search import main
    argv = ["--benchmark-folder", folder, "--searches-in-flight", str(window), "--search-batch", "16",
            "--trajectory-json", str(tmp_path / "traj.json")] + ARGS
    main(argv, vsm=tiny_vsm)             # first run of this window: engine workspaces and graphs for its batch shapes
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    records = main(argv, vsm=tiny_vsm)
    torch.cuda.synchronize()
    after = torch.cuda.memory_allocated()
    assert tiny_vsm._resident == {}
    assert after - before <= MEMORY_SLACK, (before, after)
    assert len(records) == len(alone) == N_TARGETS
    for r in records:
        a = alone[(r["test_type"], r["image"], r["target_index"])]
        assert r["expanded"] == a["expanded"]                      # boxes, bit-equal priorities, cue strings, in order
        assert (r["search_successful"], r["path_length"], r["final_box"]) == (a["search_successful"], a["path_length"], a["final_box"])
    assert any(e["context_cue"] for r in records for e in r["expanded"])           # the weak-cue branch was taken
    assert len({len(r["expanded"]) for r in records}) >= 2                       # searches of different lengths were mixed
