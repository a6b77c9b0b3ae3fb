"""TEST INFRASTRUCTURE ONLY: writes tests/golden/search_eval_golden.json from the REFERENCE's own search-only evaluation.

Run where a checkout of the reference is available (oracle/ref_shims.py, VSTAR_REFERENCE_ROOT):

    python -m tools.make_search_eval_golden

It runs the reference's `main([...])` (visual_search.py:520-564) on the synthetic tree of
tests/search_eval_helpers.make_search_bench_folder, with `VSM` replaced by tests.search_eval_helpers.SearchEvalStub and
the module's spaCy pipeline by tests.helpers.FakeNLP, and records:
  * the two lines it prints;
  * per target: success flag, path length, final patch, detection box (patch and image coordinates), IoU, and the expanded
    nodes (boxes, scores, context cues), captured by wrapping the reference module's `visual_search` and
    `visualize_search_path`;
  * the names of the files `--visualization` writes.
"""
import contextlib
import io
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_shims, vsm_oracle as O  # noqa: E402
from oracle.make_golden import GOLDEN_DIR, hf_cfgs  # noqa: E402
from tests.helpers import FakeNLP  # noqa: E402
from tests.search_eval_helpers import ARGS, SearchEvalStub, make_search_bench_folder  # noqa: E402

GOLD = os.path.join(GOLDEN_DIR, "search_eval_golden.json")


def main():
    assert ref_shims.reference_available(), "needs a checkout of the reference (VSTAR_REFERENCE_ROOT)"
    ref_shims.install(*hf_cfgs(O.tiny_config()))
    import visual_search as RVS   # the reference module
    RVS.nlp = FakeNLP()
    RVS.VSM = lambda args: SearchEvalStub()
    samples, paths = [], {}
    ref_search, ref_vis = RVS.visual_search, RVS.visualize_search_path

    def vis(image, search_path, search_length, target_bbox, label, save_path):
        paths[save_path] = [dict(bbox=[int(v) for v in s["bbox"]], score=None if s["score"] is None else float(s["score"]),
                                 context_cue=s.get("context_cue")) for s in search_path]
        return ref_vis(image, search_path, search_length, target_bbox, label, save_path)

    def search(vsm, image, target_object_name, target_bbox, smallest_size, **kw):
        fs, pl, ok, av = ref_search(vsm, image, target_object_name, target_bbox, smallest_size, **kw)
        box = fs["detection_result"].clone()          # main shifts the returned box in place afterwards
        patch = [int(v) for v in fs["bbox"]]
        img_box = box.clone()
        img_box[0] += patch[0]
        img_box[1] += patch[1]
        rel = os.path.relpath(kw["save_path"], out_root)
        test_type, stem_i = rel.split(os.sep)
        stem, i = stem_i.rsplit("_", 1)
        samples.append(dict(test_type=test_type, image=stem + ".png", target_index=int(i), target=target_object_name,
                            gt_bbox=target_bbox, smallest_size=smallest_size, search_successful=bool(ok), path_length=int(pl),
                            final_patch=patch, detection_result=box.tolist(), final_box=img_box.tolist(),
                            iou=float(RVS.iou(img_box, target_bbox)), expanded=paths.pop(kw["save_path"])))
        return fs, pl, ok, av

    RVS.visual_search, RVS.visualize_search_path = search, vis
    with tempfile.TemporaryDirectory() as tmp:
        folder = make_search_bench_folder(os.path.join(tmp, "bench"))
        out_root = os.path.join(tmp, "vis")
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            RVS.main(["--benchmark-folder", folder, "--visualization", "--output_path", out_root] + ARGS)
        files = sorted(os.path.relpath(os.path.join(d, f), out_root) for d, _, fs in os.walk(out_root) for f in fs)
    samples.sort(key=lambda s: (s["test_type"], s["image"], s["target_index"]))     # os.listdir order is file-system dependent
    gold = dict(args=ARGS, lines=buf.getvalue().splitlines(), samples=samples, visualization_files=files)
    with open(GOLD, "w") as f:
        json.dump(gold, f, indent=1)
    print("\n".join(gold["lines"]))
    print(f"{len(samples)} targets, {len(files)} visualisation files -> {GOLD}")


if __name__ == "__main__":
    main()
