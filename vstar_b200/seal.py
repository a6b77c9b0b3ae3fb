"""One V*Bench sample through the whole SEAL loop — the caller of the hot path (SURVEY.md §8f-4):
free-form answer -> "missing objects" -> guided visual search for each -> object crops -> option scoring.
Same per-sample logic and result keys as `eval_model` (/root/reference/vstar_bench_eval.py:186-273); the searches for all
missing objects of an image run in lock-step so their crop frontiers share GPU batches (the reference runs them one after
another, vstar_bench_eval.py:208-211).

Open-ended questions (the reference demo's `inference()`, app.py:130-233, below its Gradio UI): answer_open /
answer_open_many (three phases) / answer_open_stream (one pipeline), and the command line `python -m vstar_b200.seal`.
"""
from __future__ import annotations

from collections import deque
from copy import deepcopy

import numpy as np
import torch

from .visual_search import SearchController, SearchState, visual_search_many

MISSING_OBJECTS_MSG = ("Sorry, I can not answer the question. Some visual information about the following objects is missing or "
                       "unclear:")
FOCUS_MSG = "Additional visual information to focus on: "


def expand2square_center(pil_img, background_color):
    """vstar_bench_eval.py:25-36: CENTRED padding (the VSM wrapper pads bottom/right instead)"""
    from PIL import Image
    width, height = pil_img.size
    if width == height:
        return pil_img, 0, 0
    side = max(width, height)
    result = Image.new(pil_img.mode, (side, side), background_color)
    left, top = (side - width) // 2, (side - height) // 2
    result.paste(pil_img, (left, top))
    return result, left, top


def normalize_bbox(bbox, image_width, image_height):
    nb = [bbox[0] / image_width, bbox[1] / image_height, (bbox[0] + bbox[2]) / image_width, (bbox[1] + bbox[3]) / image_height]
    return [np.clip(v, 0, 1) for v in nb]


def parse_missing_objects(prediction):
    if MISSING_OBJECTS_MSG not in prediction:
        return []
    tail = prediction.split(MISSING_OBJECTS_MSG)[-1]
    if tail.endswith("."):
        tail = tail[:-1]
    return [t.strip() for t in tail.split(",")]


def focus_message(object_names, norm_boxes):
    """vstar_bench_eval.py:240-246 / app.py:198-204: the focus message over the located objects' normalised boxes"""
    msg = FOCUS_MSG
    for i, (name, b) in enumerate(zip(object_names, norm_boxes)):
        msg += "{} <object> at location [{:.3f},{:.3f},{:.3f},{:.3f}]".format(name, b[0], b[1], b[2], b[3])
        msg += "; " if i != len(norm_boxes) - 1 else "."
    return msg


def focus_question(question, object_names, norm_boxes):
    return focus_message(object_names, norm_boxes) + "\n" + question


def smallest_size_for(image, minimum_size_scale=4.0, minimum_size=224):
    """vstar_bench_eval.py:210"""
    return max(int(np.ceil(min(image.width, image.height) / minimum_size_scale)), minimum_size)


def collect_search_results(missing, results):
    """vstar_bench_eval.py:212-225: boxes of the final patch shifted to image coordinates, one entry per found instance"""
    search_result = []
    for name, (final_step, _path_length, _ok, all_valid) in zip(missing, results):
        patch = final_step["bbox"]
        boxes = all_valid if all_valid is not None else [final_step["detection_result"]]
        for b in boxes:
            b = b.clone()
            b[0] += patch[0]
            b[1] += patch[1]
            search_result.append({"bbox": b.tolist(), "name": name})
    return search_result


def choose_option(vqa_llm, image, question, options, missing, search_result):
    """vstar_bench_eval.py:226-257: option scoring, with the searched objects spliced in as <object> features"""
    return vqa_llm.multiple_choices_inference(*option_request(vqa_llm, image, question, options, missing, search_result))


def choose_options(vqa_llm, samples):
    """choose_option for several samples [(image, question, options, missing, search_result)]: one batched option scoring when
    the VQA LLM offers it (`multiple_choices_inference_batch`), the reference's one-at-a-time calls otherwise"""
    reqs = [option_request(vqa_llm, *s) for s in samples]
    if hasattr(vqa_llm, "multiple_choices_inference_batch") and len(reqs) > 1:
        return vqa_llm.multiple_choices_inference_batch(reqs)
    return [vqa_llm.multiple_choices_inference(*r) for r in reqs]


def option_request(vqa_llm, image, question, options, missing, search_result):
    """-> the argument tuple (image, question, options, object_crops, images_long, objects_long) of multiple_choices_inference"""
    if not missing:
        # the reference scores the options on the re-opened, UNPADDED image here (vstar_bench_eval.py:227, :257)
        return (image, question, options, None, None, None)
    names = [r["name"] for r in search_result]
    boxes = deepcopy([r["bbox"] for r in search_result])
    objects_long = [True] * len(names) if len(names) <= 2 else [False] * len(names)
    side = max(image.width, image.height)
    left, top = (side - image.width) // 2, (side - image.height) // 2          # expand2square (vstar_bench_eval.py:25-36)
    shifted = [[b[0] + left, b[1] + top, b[2], b[3]] for b in boxes]
    nboxes = [normalize_bbox(b, side, side) for b in shifted]
    if getattr(vqa_llm, "_img_src", None) is not None:
        # padded image + object crops cut and resized on the GPU from the resident search image (bit-identical pixels)
        padded, crops = vqa_llm.device_pixels(image, boxes, patch_scale=1.2)
    else:
        bg = tuple(int(x * 255) for x in vqa_llm.image_processor.image_mean)
        padded, _, _ = expand2square_center(image, bg)
        crops = torch.stack([vqa_llm.get_object_crop(image, b, patch_scale=1.2) for b in boxes], 0)
    return (padded, focus_question(question, names, nboxes), options, crops, [False], objects_long)


def seal_answer(vqa_llm, vsm, image, question, options, minimum_size_scale=4.0, minimum_size=224, search_batch=16,
                prediction_override=None, search_kwargs=None):
    """-> dict with the reference's per-sample result keys (question, options, prediction_freeform, missing_objects,
    search_result, option_chosen)"""
    bg = tuple(int(x * 255) for x in vqa_llm.image_processor.image_mean)
    padded, _, _ = expand2square_center(image, bg)
    prediction = prediction_override if prediction_override is not None else vqa_llm.free_form_inference(padded, question)
    missing = parse_missing_objects(prediction)
    search_result = []
    if missing:
        smallest = smallest_size_for(image, minimum_size_scale, minimum_size)
        jobs = [(image, name, smallest) for name in missing]
        results, _ = visual_search_many(vsm, jobs, batch_size=search_batch, **(search_kwargs or {}))
        search_result = collect_search_results(missing, results)
    chosen = choose_option(vqa_llm, image, question, options, missing, search_result)
    return dict(question=question, options=options, prediction_freeform=prediction, missing_objects=missing,
                search_result=search_result, option_chosen=chosen, correct=1 if chosen == 0 else 0)


# ------------------------------------------------------------------------------------------------------------------------
# open-ended questions (app.py:130-233)
OPEN_MAX_NEW_TOKENS = 512          # both generations of app.py's inference()
OPEN_CONFIDENCE_LOW = 0.3
NEED_SEARCH_MSG = "Need to conduct visual search to search for: {}."


def open_focus_question(question, object_names, norm_boxes, failed_objects, last_name):
    """app.py:198-213: the focus message over the located boxes, then one "not existent" clause per failed search.  That clause
    formats `last_name` (app.py's leaked loop variable `object_name`), not the failed object's name - kept as the reference
    prompts its model."""
    msg = focus_message(object_names, norm_boxes)
    if failed_objects:
        if object_names:
            msg = msg[:-1] + "; "
        for i, _failed in enumerate(failed_objects):
            msg += "{} not existent in the image".format(last_name)
            msg += "; " if i != len(failed_objects) - 1 else "."
    return msg + "\n" + question


def open_final_request(vqa_llm, image, question, missing, results):
    """everything app.py:158-215 computes between the searches and the final answer.  results: visual_search's
    (final_step, path_length, success, all_valid_boxes) per missing object.
    -> (final free_form_inference item (padded image, focused question, object crops, images_long, objects_long),
        search-summary string, annotated image)"""
    from .visualize import visualize_bbox
    search_result = collect_search_results(missing, results)
    failed = [name for name, (_, _, ok, _) in zip(missing, results) if not ok]
    names = [r["name"] for r in search_result]
    boxes = deepcopy([r["bbox"] for r in search_result])
    annotated = np.array(image).copy()
    for name, b in zip(names, boxes):
        annotated = visualize_bbox(annotated, b, class_name=name, color=(255, 0, 0))
    images_long = [False]
    objects_long = [True] * len(names) if len(names) <= 2 else [False] * len(names)
    crops = torch.stack([vqa_llm.get_object_crop(image, b, patch_scale=1.2) for b in boxes], 0) if boxes else None
    bg = tuple(int(x * 255) for x in vqa_llm.image_processor.image_mean)
    padded, left, top = expand2square_center(image, bg)
    nboxes = [normalize_bbox([b[0] + left, b[1] + top, b[2], b[3]], padded.width, padded.height) for b in boxes]
    last_name = names[-1] if names else missing[-1]
    q = open_focus_question(question, names, nboxes, failed, last_name)
    summary = ""
    if names:
        summary += "Targets located after search: {}.".format(", ".join(names))
    if failed:
        summary += "Targets unable to locate after search: {}.".format(", ".join(failed))
    return (padded, q, crops, images_long, objects_long), summary, annotated


def answer_open_many(vqa_llm, vsm, items, slots=16, searches_in_flight=8, minimum_size_scale=4.0, minimum_size=224, search_batch=16,
                     search_kwargs=None, temperature=0, top_p=None, num_beams=1, kv_pages=None, kv_swap_pages=None,
                     prefill_chunk=None):
    """app.py's inference() for many (image, question) pairs (PIL images), in three phases:
      A. every direct answer on one decode stream (vqa_llm.free_form_inference_stream, `slots` answers decoding at a time);
      B. every missing object's search on one SearchController.stream, `searches_in_flight` searches at a time;
      C. every final answer on one decode stream.
    temperature / top_p (sampling) and num_beams (beam search, num_beams slots per answer) apply to both decode phases, as
    free_form_inference takes them; the defaults decode greedily, as app.py does.  kv_pages = N runs both decode phases on a
    paged stream whose KV pool holds N pages (VQAEngine.decode_stream), so more answers fit in the same memory; kv_swap_pages = M
    (with kv_pages) lets an answer take pages as it writes them, preempting answers to a pinned host area of M pages when the
    pool runs dry.  prefill_chunk = C (with kv_pages) prefills admitted prompts C rows per step alongside the running answers
    (DecodeStream), so admissions stop stalling them.
    -> per item, in input order, app.py's four outputs: (direct answer, None, None, None) when nothing is missing, else
    ("Need to conduct visual search to search for: ...", search-summary string, annotated np.ndarray image, final answer)."""
    # only settings that differ from greedy are passed on, so a VQA LLM with the greedy-only signature still serves the default
    gen = {k: v for k, v, d in (("temperature", temperature, 0), ("top_p", top_p, None), ("num_beams", num_beams, 1), ("kv_pages", kv_pages, None),
                                           ("kv_swap_pages", kv_swap_pages, None), ("prefill_chunk", prefill_chunk, None))
           if v != d}
    items = [(image.convert("RGB"), question) for image, question in items]
    bg = tuple(int(x * 255) for x in vqa_llm.image_processor.image_mean)
    first = [(expand2square_center(image, bg)[0], q, None, None, None) for image, q in items]
    direct = [None] * len(items)
    for i, text in vqa_llm.free_form_inference_stream(first, max_new_tokens=OPEN_MAX_NEW_TOKENS, slots=slots, **gen):
        direct[i] = text
    missing = [parse_missing_objects(p) for p in direct]
    states, owner = [], []
    for i, (image, _) in enumerate(items):
        smallest = smallest_size_for(image, minimum_size_scale, minimum_size)
        for name in missing[i]:
            states.append(SearchState(image, name, smallest, confidence_low=OPEN_CONFIDENCE_LOW, **(search_kwargs or {})))
            owner.append(i)
    found = {}
    if states:
        ctl = SearchController(vsm, None, search_batch)
        for st, res in ctl.stream(states, window=searches_in_flight):
            found[id(st)] = res
    per_item = [[] for _ in items]
    for st, i in zip(states, owner):
        per_item[i].append(found[id(st)])
    out = [None] * len(items)
    finals, where = [], []
    for i, (image, question) in enumerate(items):
        if not missing[i]:
            out[i] = (direct[i], None, None, None)
            continue
        req, summary, annotated = open_final_request(vqa_llm, image, question, missing[i], per_item[i])
        finals.append(req)
        where.append(i)
        out[i] = [NEED_SEARCH_MSG.format(", ".join(missing[i])), summary, annotated, None]
    if finals:
        for k, text in vqa_llm.free_form_inference_stream(finals, max_new_tokens=OPEN_MAX_NEW_TOKENS, slots=slots, **gen):
            out[where[k]][3] = text
    return [tuple(o) for o in out]


def answer_open_stream(vqa_llm, vsm, items, slots=16, searches_in_flight=8, minimum_size_scale=4.0, minimum_size=224, search_batch=16,
                       search_kwargs=None, temperature=0, top_p=None, num_beams=1, kv_pages=None, kv_swap_pages=None,
                       prefill_chunk=None):
    """answer_open_many as a pipeline in which each question moves through app.py's stages on its own: its missing objects'
    searches start when its direct answer ends, and its final answer is admitted when its last search ends.  Yields
    (index, outputs) as each question completes; outputs are answer_open_many's four for that item, made by the same code.

    One host loop drives one answer session (vqa_llm.answer_session: direct and final answers share one decode stream of
    min(slots, len(items) * num_beams) slots) and one search session (SearchController.session, `searches_in_flight` searches
    at a time), on the current CUDA stream.  Each pass admits the final answers that are ready, in the order their last search
    ended, then (when none waits) direct answers in item order, while the session's admission rule allows; runs one decode
    step if an answer is running; and runs one search step if a search is active or queued.  The keywords are
    answer_open_many's.  Since the final prompts are not known when the stream opens, it holds engine.MAX_POSITIONS positions
    per request: a contiguous stream (kv_pages None) takes about 1.6 GB per slot at 7B, kv_pages bounds the pool instead.  A
    request the pool (or swap area) cannot hold raises ValueError naming its question before any launch for it; the session
    is closed then, as it is when the caller stops early.

    Sampling (temperature > 0): two seeds per item are drawn from torch's default generator before the first admission, in
    item order (direct answer, final answer), so torch.manual_seed(s) reproduces a call.  answer_open_many draws the direct
    answers' seeds and the final answers' seeds in two separate batches, so sampled answers differ between the two."""
    items = [(image.convert("RGB"), question) for image, question in items]
    if not items:
        return
    n = len(items)
    settings = None
    if (temperature is not None and temperature > 0) or num_beams != 1:
        settings = vqa_llm._stream_settings(2 * n, temperature, top_p, num_beams)
    bg = tuple(int(x * 255) for x in vqa_llm.image_processor.image_mean)
    searches = SearchController(vsm, None, search_batch).session(searches_in_flight)
    answers = vqa_llm.answer_session(OPEN_MAX_NEW_TOKENS, min(slots, n * num_beams), num_beams=num_beams, kv_pages=kv_pages,
                                     kv_swap_pages=kv_swap_pages, prefill_chunk=prefill_chunk)

    def prompt(i, item):
        p = answers.request(item)
        answers.refuse([p], f"the answer to question {i} ({items[i][1]!r})")
        return p

    def admit(i, p, stage):                 # stage 0: direct answer, 1: final answer
        answers.admit((i, stage), p, **({} if settings is None else settings[2 * i + stage]))

    try:
        ready = deque()                     # (index, final prompt) in the order their last search ended
        searching = {}                      # index -> (missing objects, their search results so far)
        finishing = {}                      # index -> its first three outputs while its final answer runs
        nxt, direct, completed = 0, None, 0
        while completed < n:
            while ready and answers.fits(ready[0][1]):
                admit(*ready.popleft(), 1)
            while not ready and nxt < n:
                if direct is None:
                    image, question = items[nxt]
                    direct = prompt(nxt, (expand2square_center(image, bg)[0], question, None, None, None))
                if not answers.fits(direct):
                    break
                admit(nxt, direct, 0)
                nxt, direct = nxt + 1, None
            if answers.busy:
                for (i, stage), text in answers.step():
                    missing = parse_missing_objects(text) if stage == 0 else None
                    if not missing:
                        completed += 1
                        yield i, (finishing.pop(i) + (text,) if stage == 1 else (text, None, None, None))
                        continue
                    image = items[i][0]
                    smallest = smallest_size_for(image, minimum_size_scale, minimum_size)
                    searching[i] = (missing, [None] * len(missing))
                    for j, name in enumerate(missing):
                        st = SearchState(image, name, smallest, confidence_low=OPEN_CONFIDENCE_LOW, **(search_kwargs or {}))
                        st.owner = (i, j)
                        searches.add(st)
            if not searches.idle:
                for st, res in searches.step():
                    i, j = st.owner
                    missing, results = searching[i]
                    results[j] = res
                    if all(r is not None for r in results):
                        del searching[i]
                        image, question = items[i]
                        req, summary, annotated = open_final_request(vqa_llm, image, question, missing, results)
                        finishing[i] = (NEED_SEARCH_MSG.format(", ".join(missing)), summary, annotated)
                        ready.append((i, prompt(i, req)))
    finally:
        answers.close()


def answer_open(vqa_llm, vsm, image, question, minimum_size_scale=4.0, minimum_size=224, **kw):
    """app.py:130-233 `inference()` below the UI for one PIL image and question -> its four outputs (see answer_open_many)"""
    return answer_open_many(vqa_llm, vsm, [(image, question)], minimum_size_scale=minimum_size_scale, minimum_size=minimum_size, **kw)[0]


def build_parser():
    """app.py's model flags (parse_args_vqallm, app.py:40-48), bench_eval's dtype / NF4 flags and the questions to answer"""
    import argparse
    p = argparse.ArgumentParser(description="SEAL open-ended answering: direct answer, visual search for the missing objects, "
                                            "final answer (the reference demo's inference(), without its web UI)")
    p.add_argument("--vqa-model-path", type=str, default="craigwu/seal_vqa_7b")
    p.add_argument("--vqa-model-base", type=str, default=None)
    p.add_argument("--conv_type", default="v1", type=str)
    p.add_argument("--vsm-model-path", type=str, default="craigwu/seal_vsm_7b")
    p.add_argument("--minimum_size_scale", default=4.0, type=float)
    p.add_argument("--minimum_size", default=224, type=int)
    p.add_argument("--vqa-dtype", default="bf16", choices=("bf16", "fp16"))
    p.add_argument("--vqa-load-4bit", action="store_true")
    q = p.add_mutually_exclusive_group(required=True)
    q.add_argument("--image", type=str, help="one image (with --question)")
    q.add_argument("--questions", type=str, help='JSONL file, one {"image": path, "question": str} per line')
    p.add_argument("--question", type=str)
    p.add_argument("--output-path", type=str, default="seal_answers.json")
    p.add_argument("--save-images", type=str, default=None, help="directory for the annotated search-result images")
    p.add_argument("--slots", default=16, type=int, help="answers decoding at a time")
    p.add_argument("--searches-in-flight", default=8, type=int)
    p.add_argument("--search-batch", default=16, type=int, help="frontier crops per VSM call")
    p.add_argument("--temperature", default=0, type=float, help="> 0: sample the answers (app.py's default 0 decodes greedily)")
    p.add_argument("--top_p", default=None, type=float, help="nucleus filter of sampled answers")
    p.add_argument("--num_beams", default=1, type=int, help="> 1: beam-search the answers (num_beams slots per answer)")
    p.add_argument("--kv-pages", default=None, type=int,
                   help="hold the answers' KV cache in a pool of this many 64-row pages, each answer reserving only the rows it needs "
                        "(default: one full-length cache slot per answer)")
    p.add_argument("--kv-swap-pages", default=None, type=int,
                   help="with --kv-pages: answers take pages as they write them, and when the pool runs dry the newest answer is "
                        "swapped to a pinned host area of this many pages until pages free (default: reserve every answer's pages "
                        "at admission)")
    p.add_argument("--prefill-chunk", default=None, type=int,
                   help="with --kv-pages: prefill admitted prompts this many rows per decode step, alongside the running answers "
                        "(default: prefill each prompt on its own at admission)")
    p.add_argument("--pipeline", action="store_true",
                   help="answer through answer_open_stream: each question's searches start when its direct answer ends and its final "
                        "answer when its searches end, direct and final answers sharing one decode stream (default: three phases, "
                        "answer_open_many)")
    return p


def read_questions(args):
    """-> [(image path, question)] from --image/--question or the --questions JSONL file"""
    import json
    if args.image is not None:
        if not args.question:
            raise SystemExit("--image needs --question")
        return [(args.image, args.question)]
    out = []
    with open(args.questions) as f:
        for line in f:
            if line.strip():
                rec = json.loads(line)
                out.append((rec["image"], rec["question"]))
    return out


def write_answers(path, questions, answers, save_images=None):
    """one JSON record per question: image, question, direct_answer, search_summary, final_answer, annotated_image"""
    import json
    import os
    recs = []
    for k, ((img_path, question), (a0, a1, a2, a3)) in enumerate(zip(questions, answers)):
        rec = dict(image=img_path, question=question, direct_answer=a0, search_summary=a1, final_answer=a3, annotated_image=None)
        if a2 is not None and save_images:
            from PIL import Image
            os.makedirs(save_images, exist_ok=True)
            rec["annotated_image"] = os.path.join(save_images, f"{k:05d}_search_result.png")
            Image.fromarray(a2).save(rec["annotated_image"])
        recs.append(rec)
    with open(path, "w") as f:
        json.dump(recs, f, indent=1)
    return recs


def main(argv=None, vqa_llm=None, vsm=None):
    from PIL import Image
    args = build_parser().parse_args(argv)
    questions = read_questions(args)
    if vqa_llm is None:
        from .vqa import VQA_LLM
        vqa_llm = VQA_LLM(args)
    if vsm is None:
        from .visual_search import parse_args
        from .vsm import VSM
        vsm_args = parse_args({})
        vsm_args.version = args.vsm_model_path
        vsm = VSM(vsm_args)
    items = [(Image.open(p).convert("RGB"), q) for p, q in questions]
    kw = dict(slots=args.slots, searches_in_flight=args.searches_in_flight, minimum_size_scale=args.minimum_size_scale,
              minimum_size=args.minimum_size, search_batch=args.search_batch, temperature=args.temperature, top_p=args.top_p,
              num_beams=args.num_beams, kv_pages=args.kv_pages, kv_swap_pages=args.kv_swap_pages, prefill_chunk=args.prefill_chunk)
    if args.pipeline:
        answers = [None] * len(items)
        for i, out in answer_open_stream(vqa_llm, vsm, items, **kw):
            answers[i] = out
    else:
        answers = answer_open_many(vqa_llm, vsm, items, **kw)
    return write_answers(args.output_path, questions, answers, args.save_images)


if __name__ == "__main__":
    main()
