"""Test-only fixtures for the search-only V*Bench evaluation (`vstar_b200.visual_search.main`, reference visual_search.py:520-564):
a small synthetic benchmark tree whose targets cover every outcome of a search, and the stub VSM it is searched with.
The golden tests/golden/search_eval_golden.json is the reference's own `main` run on this tree with this stub
(tools/make_search_eval_golden.py)."""
import json
import os

import numpy as np

from tests.helpers import RecordStub, StubVSM, synth_image

# the arguments every run of the tree uses: leaves stop at min side <= 320, so with the stub's "small" mode (confident only on
# crops whose min side is <= 300) an image can be searched to the bottom without a confident hit; the cue thresholds sit inside
# the stub's heat-map range, so some nodes take the weak-cue branch and others do not
ARGS = ["--minimum_size", "320", "--target_cue_threshold", "11.0", "--target_cue_threshold_decay", "0.95",
        "--target_cue_threshold_minimum", "10.0"]


def dim_dark_crop(image, logits):
    """detection scores of a dark crop (mean pixel value below 64) quartered: 0.45 at most, under confidence_low"""
    if logits is not None and float(np.asarray(image, dtype=np.uint8).mean()) < 64:
        return logits * 0.25
    return logits


class SearchEvalStub(StubVSM):
    """StubVSM(hot="small") that never finds anything on a dark image, not even through the confidence_low fallback, so the
    tree also has failed searches.  Still a pure function of the crop's pixels and the question."""

    def __init__(self):
        super().__init__("small")

    def _eval(self, image, question, mode):
        ans, boxes, logits, low = super()._eval(image, question, mode)
        return ans, boxes, dim_dark_crop(image, logits), low


class SearchEvalRecordStub(RecordStub):
    """the same function through the batched launch / finish record interface of the CUDA VSM"""

    def __init__(self):
        super().__init__("small")

    def _eval(self, image, question, mode):
        ans, boxes, logits, low = super()._eval(image, question, mode)
        return ans, boxes, dim_dark_crop(image, logits), low


def dark_image(seed, w, h):
    from PIL import Image
    return Image.fromarray(np.random.default_rng(seed).integers(0, 60, (h, w, 3), dtype=np.uint8), "RGB")


# (name, seed, w, h, dark, [(gt_bbox, target_object)]).  Outcomes with ARGS and SearchEvalStub:
#   se_root   280x200    confident at the root (path length 1)
#   se_deep   1000x800   confident on the fourth node, three levels down, after weak-cue nodes
#   se_wide   1400x330   4x1 split at the root, confident on the third node
#   se_fall   330x310    root is the smallest unit and never confident: success through the confidence_low fallback
#   se_full   1240x1240  the whole 21-node tree without a confident hit (some weak-cue nodes), then the confidence_low fallback
#   se_dark   330x310    dark: nothing passes confidence_low (failed search)
#   se_dark2  700x650    dark: the whole 21-node tree, failed
SPEC = {
    "direct_attributes": [
        ("se_root", 51, 280, 200, False, [([200.0, 30.0, 40.0, 145.0], "mug")]),
        ("se_deep", 52, 1000, 800, False, [([0.0, 280.0, 195.0, 82.0], "red mug"), ([10, 10, 50, 50], "kettle")]),
        ("se_fall", 53, 330, 310, False, [([20, 30, 100, 80], "lamp")]),
        ("se_dark", 54, 330, 310, True, [([0, 0, 40, 40], "dog"), ([100, 100, 60, 60], "cup")]),
    ],
    "relative_position": [
        ("se_wide", 55, 1400, 330, False, [([60.0, 175.0, 35.0, 95.0], "sign"), ([20, 20, 30, 30], "tree"),
                                           ([1200, 200, 90, 80], "car")]),
        ("se_full", 56, 1240, 1240, False, [([760.0, 570.0, 455.0, 385.0], "chair")]),
        ("se_dark2", 57, 700, 650, True, [([10, 10, 100, 100], "door"), ([300, 300, 80, 80], "bed")]),
    ],
}


def make_search_bench_folder(root, spec=None):
    """synthetic V*Bench tree for the search-only evaluation: <root>/{direct_attributes,relative_position}/{name}.png + {name}.json
    with the annotation keys the evaluation reads (`bbox`, `target_object`) next to a question, as in V*Bench"""
    for test_type, items in (spec or SPEC).items():
        d = os.path.join(root, test_type)
        os.makedirs(d, exist_ok=True)
        for name, seed, w, h, dark, targets in items:
            (dark_image if dark else synth_image)(seed, w, h).save(os.path.join(d, name + ".png"))
            with open(os.path.join(d, name + ".json"), "w") as f:
                json.dump({"question": f"Where is the {targets[0][1]}?", "bbox": [list(b) for b, _ in targets],
                           "target_object": [t for _, t in targets]}, f)
    return root
