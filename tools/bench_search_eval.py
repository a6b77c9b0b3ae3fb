"""Search-only V*Bench evaluation (`python -m vstar_b200.visual_search`) at full size: how much the window of searches in flight
(--searches-in-flight W) buys over the reference's one-search-at-a-time schedule (W = 1).

Workload: a synthetic V*Bench-shaped tree written to a temporary directory: 64 JPEG images around V*Bench's typical
2246 x 1582, 1 or 2 targets each, searched with the full-size VSM (Vicuna-7B / CLIP-L / OWL-ViT-B / SAM-decoder shapes,
random bf16 weights) and the forced "[LOC]" answer that bench.py uses.  Random weights give no real detections, so
--confidence_high is set to the 92nd percentile of the root-and-below crop scores of a calibration search: about one crop in
twelve ends its search, and search lengths spread from the root alone to the whole 21-node tree like they do on V*Bench.
The cue thresholds are the reference's defaults.

Each W runs the whole tree through `main`, the settings alternating (1, 8, 32, 1, 8, 32, ...) after a warm-up that
runs every W on a small tree and the largest W once on the measured tree.  Per run:
searches/s, crops/s (crops launched on the GPU, speculative ones included, and crops committed to a search), median and p90
of per-search latency (admission to finish).  The per-target results of every run are checked to be identical.  The GPU
name, power limit and max SM clock are read in the same run.

    python tools/bench_search_eval.py [--images 64] [--rounds 2] [--windows 1,8,32] [--out bench_out/search_eval]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from PIL import Image

NAMES = ("mug", "dog", "red car", "traffic light", "umbrella", "backpack", "bicycle", "clock")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().split("\n")[0]
    except (OSError, subprocess.SubprocessError):
        q = ""
    return dict(device=torch.cuda.get_device_name(), nvidia_smi=q)


def make_tree(root, n_images, seed=0):
    """V*Bench-shaped tree: images split over the two test types, sizes around 2246 x 1582, 1 or 2 targets each"""
    rng = np.random.default_rng(seed)
    for k in range(n_images):
        test_type = "direct_attributes" if k < (n_images * 3) // 5 else "relative_position"
        d = os.path.join(root, test_type)
        os.makedirs(d, exist_ok=True)
        w, h = int(2246 + rng.integers(-160, 161)), int(1582 + rng.integers(-120, 121))
        if rng.random() < 0.25:
            w, h = h, w                                    # some portrait images
        # smooth colour field plus noise: JPEG sizes and decode times in the range of photographs
        base = rng.integers(0, 256, (h // 32 + 1, w // 32 + 1, 3), dtype=np.uint8)
        img = Image.fromarray(base).resize((w, h), Image.BILINEAR)
        arr = np.asarray(img, dtype=np.int16) + rng.integers(-24, 25, (h, w, 3), dtype=np.int16)
        Image.fromarray(np.clip(arr, 0, 255).astype(np.uint8)).save(os.path.join(d, f"sa_{k}.jpg"), quality=90)
        n_t = 1 + int(rng.random() < 0.5)
        boxes = [[int(rng.integers(0, w - 200)), int(rng.integers(0, h - 200)), int(rng.integers(20, 200)), int(rng.integers(20, 200))]
                 for _ in range(n_t)]
        names = [NAMES[int(i)] for i in rng.choice(len(NAMES), n_t, replace=False)]
        with open(os.path.join(d, f"sa_{k}.json"), "w") as f:
            json.dump({"question": f"What is the color of the {names[0]}?", "options": ["red", "blue"], "bbox": boxes,
                       "target_object": names}, f)
    return root


def build_vsm(tiny, batch):
    from vstar_b200 import synth
    from vstar_b200.config import VSMConfig, tiny_config
    from vstar_b200.engine import VSMEngine, VSMWeights
    from vstar_b200.vsm import VSM
    cfg = tiny_config() if tiny else VSMConfig()
    shapes = synth.state_dict_shapes(cfg)
    eng = VSMEngine(VSMWeights(cfg, lambda n: synth.synthetic_tensor(n, shapes[n], seed=1234, device="cuda", dtype=torch.bfloat16)),
                    max_tokens=384)
    prompt, ans = synth.synthetic_prompt(cfg, n_text=60, seed=0, im_start_index=None if tiny else 37)

    class BenchVSM(VSM):
        """synthetic tokenisation as in bench.py; counts the crops it is asked to evaluate"""
        launched = 0
        cue_crops = 0

        def _ids(self, question):
            return prompt[0].tolist()

        def detect_regions_launch(self, regions, *a, **k):
            self.launched += len(regions)
            return super().detect_regions_launch(regions, *a, **k)

        def inference_many(self, regions, *a, **k):
            self.cue_crops += len(regions)
            return super().inference_many(regions, *a, **k)

    return BenchVSM(engine=eng, forced_answer_ids=ans.tolist(), frontier_batch=batch)


def calibrate(vsm, folder, batch, q):
    """confidence_high = the q-quantile of the crop scores of full-tree searches on the first images"""
    from vstar_b200.bench_eval import TEST_TYPES, list_samples
    from vstar_b200.seal import smallest_size_for
    from vstar_b200.visual_search import visual_search_many
    imgs = [Image.open(p).convert("RGB") for _, p, _ in list_samples(os.path.join(folder, TEST_TYPES[0]))[:4]]
    jobs = [(im, "mug", smallest_size_for(im)) for im in imgs]
    _, states = visual_search_many(vsm, jobs, batch_size=batch, confidence_high=2.0)
    vsm.release()
    top = [ev.top_logit for st in states for ev in st.cache.values() if ev.top_logit is not None]
    return float(np.quantile(top, q)), dict(n=len(top), min=float(np.min(top)), median=float(np.median(top)), max=float(np.max(top)))


def run_once(vsm, folder, window, batch, conf, tmp):
    from vstar_b200.visual_search import main
    traj = os.path.join(tmp, f"traj_{window}.json")
    argv = ["--benchmark-folder", folder, "--searches-in-flight", str(window), "--search-batch", str(batch),
            "--confidence_high", repr(conf), "--trajectory-json", traj]
    l0, c0, t_prep, t_eng = vsm.launched, vsm.cue_crops, vsm.timers["prep"], vsm.timers["engine"]
    torch.cuda.synchronize()
    t = time.perf_counter()
    records = main(argv, vsm=vsm)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t
    lat = np.array([r["latency_s"] for r in records])
    committed = sum(r["evaluations"] for r in records)
    out = dict(window=window, search_batch=batch, searches=len(records), wall_s=round(wall, 3),
               searches_per_s=round(len(records) / wall, 3), crops_launched=vsm.launched - l0,
               crops_launched_per_s=round((vsm.launched - l0) / wall, 2), crops_committed=committed,
               crops_committed_per_s=round(committed / wall, 2), cue_crops=vsm.cue_crops - c0,
               latency_median_s=round(float(np.median(lat)), 4), latency_p90_s=round(float(np.quantile(lat, 0.9)), 4),
               host_prep_s=round(vsm.timers["prep"] - t_prep, 3), host_engine_calls_s=round(vsm.timers["engine"] - t_eng, 3),
               resident_after=len(vsm._resident), top1_acc=json.load(open(traj))["top1_acc"])
    key = {(r["test_type"], r["image"], r["target_index"]): (r["search_successful"], r["path_length"], r["final_box"], r["expanded"])
           for r in records}
    lengths = [len(r["expanded"]) for r in records]
    return out, key, lengths


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--windows", default="1,8,32")
    ap.add_argument("--batch", type=int, default=64, help="--search-batch of every run")
    ap.add_argument("--quantile", type=float, default=0.92)
    ap.add_argument("--tiny", action="store_true", help="tiny model config (a quick check of the script, not a measurement)")
    ap.add_argument("--out", default="bench_out/search_eval")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from vstar_b200 import noun_chunks
    noun_chunks.set_nlp(lambda text: [])       # synthetic cue answers carry no parsable nouns: "region {phrase}" prompts
    windows = [int(w) for w in args.windows.split(",")]
    info = gpu_info()
    print(json.dumps(info), flush=True)
    t0 = time.perf_counter()
    vsm = build_vsm(args.tiny, args.batch)
    load_s = time.perf_counter() - t0
    with tempfile.TemporaryDirectory() as tmp:
        folder = make_tree(os.path.join(tmp, "bench"), args.images)
        warm = make_tree(os.path.join(tmp, "warm"), 6, seed=1)
        conf, scores = calibrate(vsm, warm, args.batch, args.quantile)
        print(json.dumps(dict(confidence_high=conf, calibration_scores=scores)), flush=True)
        for w in windows:                       # warm-up: every window's batch shapes, graphs and allocator growth
            run_once(vsm, warm, w, args.batch, conf, tmp)
        run_once(vsm, folder, max(windows), args.batch, conf, tmp)     # and the first touch of every image size of the tree
        runs, ref_key, lengths = [], None, None
        for rnd in range(args.rounds):
            for w in windows:
                r, key, ln = run_once(vsm, folder, w, args.batch, conf, tmp)
                r["round"] = rnd
                if ref_key is None:
                    ref_key, lengths = key, ln
                r["results_identical_to_first_run"] = key == ref_key
                runs.append(r)
                print(json.dumps(r), flush=True)
    summary = {}
    for w in windows:
        rs = [r for r in runs if r["window"] == w]
        summary[str(w)] = {k: float(np.median([r[k] for r in rs])) for k in
                           ("searches_per_s", "crops_launched_per_s", "crops_committed_per_s", "latency_median_s", "latency_p90_s", "wall_s")}
    hist = np.bincount(lengths).tolist()
    result = dict(gpu=info, model="tiny" if args.tiny else "7B shapes, random bf16 weights, forced [LOC] answer", images=args.images,
                  searches=len(lengths), search_batch=args.batch, confidence_high=conf, calibration_scores=scores,
                  search_length_histogram=hist, load_s=round(load_s, 1), runs=runs, median_over_rounds=summary,
                  all_results_identical=all(r["results_identical_to_first_run"] for r in runs))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_search_eval.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(dict(median_over_rounds=summary, all_results_identical=result["all_results_identical"])), flush=True)


if __name__ == "__main__":
    main()
