"""V*Bench driver — the caller on the far side of the hot path (SURVEY.md §8f-4).

Mirrors `eval_model` of /root/reference/vstar_bench_eval.py:168-273: same folder walk (`direct_attributes`,
`relative_position`; every non-.json file is an image whose annotation sits beside it), same per-sample logic and the same
output JSON (keys question, options, image, prediction_freeform, missing_objects, search_result, option_chosen, correct;
`json.dump(results, f, indent=4)`), same accuracy prints.

What changes is the schedule.  The reference answers one image at a time and runs the searches of that image one after
another (vstar_bench_eval.py:208-211), so the VSM sees batch 1.  Here `images_in_flight` images are taken together:
  1. free-form answers for the chunk in ONE continuous-batched greedy decode (`VQA_LLM.free_form_inference_batch`: ragged
     left-padded KV cache, every decode step reads the 7B weights once for all images) -> missing objects,
  2. ONE lock-step `visual_search_many` over every (image, missing object) of the chunk, so root and level-2 rounds, which
     cannot fill a GPU (let alone eight) on their own, share frontier batches (SURVEY.md §8e "scaling loss sources"),
  3. option scoring.
Searches are independent, so the per-sample results do not depend on the chunk size (tests/test_bench_eval.py).
"""
from __future__ import annotations

import argparse
import json
import os
from collections import defaultdict

import numpy as np

from .seal import (choose_options, collect_search_results, expand2square_center, parse_missing_objects, smallest_size_for)
from .visual_search import visual_search_many

TEST_TYPES = ("direct_attributes", "relative_position")


def build_parser():
    """argument names and defaults of vstar_bench_eval.py:275-284, plus the scheduling knobs of this implementation"""
    p = argparse.ArgumentParser()
    p.add_argument("--vqa-model-path", type=str, default="craigwu/seal_vqa_7b")
    p.add_argument("--vqa-model-base", type=str, default=None)
    p.add_argument("--conv_type", default="v1", type=str)
    p.add_argument("--benchmark-folder", type=str, default="vstar_bench")
    p.add_argument("--vsm-model-path", type=str, default="craigwu/seal_vsm_7b")
    p.add_argument("--output-path", type=str, default="eval_result.json")
    p.add_argument("--minimum_size_scale", default=4.0, type=float, help="minimum sub-image scale for the termination of search")
    p.add_argument("--minimum_size", default=224, type=int, help="minimum sub-image size for the termination of search")
    p.add_argument("--images-in-flight", default=8, type=int, help="images whose searches share GPU batches")
    p.add_argument("--search-batch", default=64, type=int, help="frontier crops per VSM call")
    p.add_argument("--vqa-dtype", default="bf16", choices=("bf16", "fp16"),
                   help="compute dtype of the SEAL VQA LLM: fp16 is the reference's (LLaVA/llava/model/builder.py:43); the VSM stays bf16")
    p.add_argument("--vqa-load-4bit", action="store_true",
                   help="load the SEAL VQA LLM's Linear weights in NF4 (the reference's load_4bit); computes in fp16 whatever --vqa-dtype says")
    return p


def list_samples(folder):
    """vstar_bench_eval.py:185-191 (os.listdir order, as the reference; annotation = image file name up to its first '.').
    The reference cuts the whole path at its first '.', which breaks under a directory with a dot in its name; only the
    file name is cut here."""
    files = [f for f in os.listdir(folder) if ".json" not in f]
    return [(f, os.path.join(folder, f), os.path.join(folder, f.split(".")[0] + ".json")) for f in files]


def eval_model(args, vqa_llm=None, vsm=None, log=print, search_kwargs=None):
    """Run the benchmark; returns (results dict, overall accuracy).  `vqa_llm` / `vsm` may be injected (tests, sharded VSM);
    otherwise they are built from `args` exactly as vstar_bench_eval.py:169-174 does."""
    from PIL import Image
    if vqa_llm is None:
        from .vqa import VQA_LLM
        vqa_llm = VQA_LLM(args)
    if vsm is None:
        from .visual_search import parse_args
        from .vsm import VSM
        vsm_args = parse_args({})
        vsm_args.version = args.vsm_model_path
        vsm = VSM(vsm_args)
    if hasattr(vqa_llm, "use_device_images") and getattr(vsm, "pipeline", None) is not None:
        vqa_llm.use_device_images(vsm)         # option-scoring pixels from the search image that is already resident in HBM
    in_flight = max(1, int(getattr(args, "images_in_flight", 8)))
    search_batch = int(getattr(args, "search_batch", 64))
    bg = tuple(int(x * 255) for x in vqa_llm.image_processor.image_mean)

    results, per_type_acc, all_acc = {}, defaultdict(list), []
    for test_type in TEST_TYPES:
        results[test_type] = []
        samples = list_samples(os.path.join(args.benchmark_folder, test_type))
        for c0 in range(0, len(samples), in_flight):
            chunk = []
            for image_file, image_path, annotation_path in samples[c0:c0 + in_flight]:
                image = Image.open(image_path).convert("RGB")
                chunk.append(dict(image_file=image_file, image=image, annotation=json.load(open(annotation_path))))
            padded = [expand2square_center(smp["image"], bg)[0] for smp in chunk]
            questions = [smp["annotation"]["question"] for smp in chunk]
            if hasattr(vqa_llm, "free_form_inference_batch") and len(chunk) > 1:
                predictions = vqa_llm.free_form_inference_batch(padded, questions, originals=[smp["image"] for smp in chunk])      # one continuous-batched decode
            else:
                predictions = [vqa_llm.free_form_inference(im, q) for im, q in zip(padded, questions)]
            for smp, prediction in zip(chunk, predictions):
                smp["prediction"] = prediction
                smp["missing"] = parse_missing_objects(prediction)
            jobs, owner = [], []
            for i, smp in enumerate(chunk):
                smallest = smallest_size_for(smp["image"], args.minimum_size_scale, args.minimum_size)
                for name in smp["missing"]:
                    jobs.append((smp["image"], name, smallest))
                    owner.append(i)
            found = [[] for _ in chunk]
            if jobs:
                search_results, _ = visual_search_many(vsm, jobs, batch_size=search_batch, **(search_kwargs or {}))
                for i, r in zip(owner, search_results):
                    found[i].append(r)
            search_results = [collect_search_results(smp["missing"], res) if smp["missing"] else [] for smp, res in zip(chunk, found)]
            chosen_all = choose_options(vqa_llm, [(smp["image"], smp["annotation"]["question"], smp["annotation"]["options"], smp["missing"], sr)
                                                  for smp, sr in zip(chunk, search_results)])       # one batched option scoring
            for smp, search_result, chosen in zip(chunk, search_results, chosen_all):
                ann = smp["annotation"]
                correct = 1 if chosen == 0 else 0
                per_type_acc[test_type].append(correct)
                all_acc.append(correct)
                results[test_type].append(dict(question=ann["question"], options=ann["options"], image=smp["image_file"],
                                               prediction_freeform=smp["prediction"], missing_objects=smp["missing"],
                                               search_result=search_result, option_chosen=chosen, correct=correct))
        log(test_type, np.mean(per_type_acc[test_type]) if per_type_acc[test_type] else float("nan"))
    overall = float(np.mean(all_acc)) if all_acc else float("nan")
    log(overall)
    with open(args.output_path, "w") as f:
        json.dump(results, f, indent=4)
    return results, overall


def main(argv=None):
    args = build_parser().parse_args(argv)
    eval_model(args)


if __name__ == "__main__":
    main()
