"""What pipelining open-ended SEAL answering (seal.answer_open_stream) buys over its three phases (seal.answer_open_many) on the
same work, with the VQA LLM and the VSM at 7B shapes (random weights), both resident, in bf16 and with the VQA LLM in NF4.

Workload: 64 synthetic images at V*Bench-like sizes (tools/bench_search_eval.make_tree), one open question each, and
--confidence_high calibrated as bench_search_eval does, so search lengths spread over the tree.  Random weights can neither
name missing objects nor stop, so two parts are scripted the same way in both arms:
  * direct answers: a seeded ~60 % of the questions name 1-3 missing objects (the text of the direct answer is replaced, as
    tests/test_vqa_stream_gpu.py's ScriptedLLM does), the rest answer directly;
  * answer lengths: every direct and final answer decodes to a length drawn log-uniformly (direct 4-128, final 16-512 tokens)
    and is ended there by a DecodeStream subclass standing in for a trained model's eos (as tools/bench_vqa_stream_swap.py
    does), keyed by the prompt so both arms end the same answer at the same length.
Both arms decode greedily on a paged stream of `slots` 16 whose pool holds the bytes of 16 contiguous slots of 2048 positions.

Per arm, alternated over --rounds rounds after a warm-up of both: wall time and questions/s; latency per question from the
admission of its direct answer to the end of its last answer on the stream (p50, p90; the phased call hands every result back
only when it returns, which the wall time shows), and the time to the first completed question; decode steps and mean rows
per step; mean frontier batch of the VSM.  Both arms are then run once in batch-invariant mode and compared item by item on all
four outputs (the first --check-items questions); the default-mode runs report how many items agree.  The GPU name, power limit and max SM clock are read in the
same run.

    python tools/bench_seal_pipeline.py [--images 64] [--rounds 2] [--dtypes bf16,nf4] [--check-items 16] [--out results.json]
(--out keeps the dtypes of earlier runs already in the file, so each dtype can run on its own)
"""
import argparse
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from PIL import Image

from tools.bench_search_eval import build_vsm, calibrate, gpu_info, make_tree
from tools.bench_vqa_stream_paged import equal_bytes_pages
from vstar_b200 import ops, seal, synth
from vstar_b200.config import VSMConfig
from vstar_b200.vqa import VQA_LLM, AnswerSession, DecodeStream, VQAEngine, VQAWeights

SLOTS = 16
POSITIONS = 2048                   # engine.MAX_POSITIONS: what one contiguous slot of the pipeline's session holds
WINDOW, SEARCH_BATCH = 8, 16       # answer_open_many's defaults
NAMES = ("mug", "dog", "red car", "traffic light", "umbrella", "backpack", "bicycle", "clock")


class Clock:
    """what both arms record: the ends drawn per prompt, admission and end times per prompt, steps and rows"""

    def __init__(self):
        self.ends, self.admitted, self.ended = {}, {}, {}
        self.steps = self.rows = 0

    def end_for(self, ids):
        key = tuple(ids)
        if key not in self.ends:                      # a final prompt: its length drawn from its ids, the same in both arms
            rng = np.random.default_rng(abs(hash(key)) % 2 ** 32)
            self.ends[key] = int(np.exp(rng.uniform(np.log(16), np.log(512))))
        return self.ends[key]


CLOCK = Clock()


class EndsAt(DecodeStream):
    """a request ends after CLOCK.end_for(its prompt) tokens (a trained model's eos, which random weights never emit); records
    admission and end times per prompt"""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self._ends, self._ids = {}, {}

    def admit(self, request, *a, **kw):
        key = tuple(request[0])
        self._ends[self._next_id], self._ids[self._next_id] = CLOCK.end_for(key), key
        CLOCK.admitted.setdefault(key, time.perf_counter())
        return super().admit(request, *a, **kw)

    def _ended(self, r):
        return len(r.tokens) >= self._ends[r.id] or super()._ended(r)

    def step(self):
        s0, o0 = self.steps, self.occupied
        done = super().step()
        CLOCK.steps += self.steps - s0
        CLOCK.rows += self.occupied - o0
        t = time.perf_counter()
        for r, _ in done:
            CLOCK.ended[self._ids[r.id]] = t
        return done


class BenchEngine(VQAEngine):
    def decode_stream(self, max_slots, max_positions=None, eos_token_id=2, temperature=0, num_beams=1, kv_pages=None, kv_swap_pages=None,
                      prefill_chunk=None):
        return EndsAt(self, max_slots, self.max_tokens if max_positions is None else max_positions, -1, kv_pages=kv_pages,
                      kv_swap_pages=kv_swap_pages, prefill_chunk=prefill_chunk)


def scripted_llm(engine, missing):
    """VQA_LLM whose direct answers name `missing[i]` (question i) on both decode paths"""
    def script(i, text):
        return seal.MISSING_OBJECTS_MSG + " " + ", ".join(missing[i]) + "." if missing[i] else text

    class ScriptedSession(AnswerSession):
        def step(self):
            return [((i, stage), script(i, text) if stage == 0 else text) for (i, stage), text in super().step()]

    class ScriptedLLM(VQA_LLM):
        def free_form_inference_stream(self, items, *a, **kw):
            for i, text in super().free_form_inference_stream(items, *a, **kw):
                q = items[i][1]
                yield i, text if seal.FOCUS_MSG in q else script(int(q.split()[1]), text)

        def answer_session(self, max_new_tokens, slots, max_positions=None, num_beams=1, **kw):
            return ScriptedSession(self, max_new_tokens, slots, max_positions or self.engine.MAX_POSITIONS, num_beams, **kw)

    return ScriptedLLM(engine=engine)


def run_arm(arm, llm, vsm, items, conf, pages, direct_ids):
    CLOCK.admitted, CLOCK.ended, CLOCK.steps, CLOCK.rows = {}, {}, 0, 0
    l0, n0 = vsm.launched, vsm.launches
    kw = dict(slots=SLOTS, searches_in_flight=WINDOW, search_batch=SEARCH_BATCH, kv_pages=pages,
              search_kwargs=dict(confidence_high=conf))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if arm == "pipelined":
        outs, done = [None] * len(items), {}
        for i, o in seal.answer_open_stream(llm, vsm, items, **kw):
            outs[i], done[i] = o, time.perf_counter()
    else:
        outs = seal.answer_open_many(llm, vsm, items, **kw)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    vsm.release()
    if arm == "phased":                  # a question is complete when its last answer ended on the stream
        done = {}
        for i in range(len(items)):
            done[i] = CLOCK.ended[direct_ids[i]] if outs[i][1] is None else None
        finals = sorted((CLOCK.admitted[k], k) for k in CLOCK.ended if k not in set(direct_ids))
        where = [i for i, o in enumerate(outs) if o[1] is not None]
        for (_, k), i in zip(finals, where):               # phase C admits the finals in item order
            done[i] = CLOCK.ended[k]
    lat = np.array([done[i] - CLOCK.admitted[direct_ids[i]] for i in range(len(items))])
    first = min(done.values()) - t0
    return outs, dict(wall_s=round(wall, 3), questions_per_s=round(len(items) / wall, 3), latency_p50_s=round(float(np.median(lat)), 3),
                      latency_p90_s=round(float(np.quantile(lat, 0.9)), 3), first_completed_s=round(first, 3), decode_steps=CLOCK.steps,
                      rows_per_step=round(CLOCK.rows / max(1, CLOCK.steps), 2),
                      search_batch_mean=round((vsm.launched - l0) / max(1, vsm.launches - n0), 2))


def keyed(outs):
    return [(o[0], o[1], None if o[2] is None else o[2].tobytes(), o[3]) for o in outs]


def bench_dtype(name, make_weights, vsm, items, missing, conf, rounds, check):
    llm = scripted_llm(BenchEngine(make_weights(), max_tokens=1536), missing)
    pages = equal_bytes_pages(SLOTS, POSITIONS)
    direct_ids = [tuple(llm._prompt_ids(q)) for _, q in items]
    rng = np.random.default_rng(7)
    for k in direct_ids:
        CLOCK.ends[k] = int(np.exp(rng.uniform(np.log(4), np.log(128))))
    for arm in ("phased", "pipelined"):                   # warm-up on the first eight questions
        run_arm(arm, llm, vsm, items[:8], conf, pages, direct_ids)
    runs, outs = [], {}
    for rnd in range(rounds):
        for arm in ("phased", "pipelined"):
            outs[arm], r = run_arm(arm, llm, vsm, items, conf, pages, direct_ids)
            runs.append(dict(r, arm=arm, round=rnd))
            print(json.dumps({name: runs[-1]}), flush=True)
    agree_default = sum(a == b for a, b in zip(keyed(outs["phased"]), keyed(outs["pipelined"])))
    with ops.batch_invariant():
        inv = {arm: run_arm(arm, llm, vsm, items[:check], conf, pages, direct_ids)[0] for arm in ("phased", "pipelined")}
    same = keyed(inv["phased"]) == keyed(inv["pipelined"])
    summary = {}
    for arm in ("phased", "pipelined"):
        rs = [r for r in runs if r["arm"] == arm]
        summary[arm] = {k: float(np.median([r[k] for r in rs])) for k in rs[0] if k not in ("arm", "round")}
        summary[arm]["wall_s_spread"] = [min(r["wall_s"] for r in rs), max(r["wall_s"] for r in rs)]
    summary["pipelined_over_phased_questions_per_s"] = round(summary["pipelined"]["questions_per_s"] / summary["phased"]["questions_per_s"], 3)
    del llm
    torch.cuda.empty_cache()
    return dict(kv_pages=pages, slots=SLOTS, runs=runs, median_over_rounds=summary, default_mode_items_agreeing=agree_default,
                batch_invariant_items_checked=check, batch_invariant_outputs_identical=same)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--dtypes", default="bf16,nf4")
    ap.add_argument("--quantile", type=float, default=0.92)
    ap.add_argument("--check-items", type=int, default=16, help="questions compared between the arms in batch-invariant mode")
    ap.add_argument("--out", default=None, help="also write the result JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_seal_pipeline needs a CUDA GPU (nothing is measured on the CPU)")
    from vstar_b200 import noun_chunks
    noun_chunks.set_nlp(lambda text: [])       # synthetic cue answers carry no parsable nouns: "region {phrase}" prompts
    res = dict(gpu_before=gpu_info(), images=a.images, rounds=a.rounds, slots=SLOTS, searches_in_flight=WINDOW, search_batch=SEARCH_BATCH)
    vsm = build_vsm(False, SEARCH_BATCH)
    vsm.launches = 0
    launch, finish = vsm.detect_regions_launch, vsm.detect_regions_finish

    def counted(*x, **k):
        vsm.launches += 1
        return launch(*x, **k)

    def at_most_two_valid(handle):
        # random weights put hundreds of boxes above 0.5 in a crop: a search that ends at its root would hand all of them to
        # the final prompt as object crops, past the 2048 positions.  A trained model finds an object or two.
        evs = finish(handle)
        for ev in evs:
            if ev.n_valid is not None and ev.n_valid > 2:
                ev.n_valid, ev.valid_boxes = 2, ev.valid_boxes[:2]
        return evs
    vsm.detect_regions_launch, vsm.detect_regions_finish = counted, at_most_two_valid
    rng = np.random.default_rng(0)
    missing = [[NAMES[int(j)] for j in rng.choice(len(NAMES), int(rng.integers(1, 4)), replace=False)] if rng.random() < 0.6 else []
               for _ in range(a.images)]
    with tempfile.TemporaryDirectory() as tmp:
        folder = make_tree(os.path.join(tmp, "bench"), a.images)
        warm = make_tree(os.path.join(tmp, "warm"), 6, seed=1)
        conf, scores = calibrate(vsm, warm, SEARCH_BATCH, a.quantile)
        from vstar_b200.bench_eval import TEST_TYPES, list_samples
        paths = [p for t in TEST_TYPES for _, p, _ in list_samples(os.path.join(folder, t))]
        items = [(Image.open(p).convert("RGB"), f"question {i} what is the colour of the {NAMES[i % len(NAMES)]}")
                 for i, p in enumerate(paths)]
    res.update(confidence_high=conf, calibration_scores=scores, questions_with_missing=sum(map(bool, missing)),
               missing_objects=sum(map(len, missing)))
    cfg = VSMConfig()
    shapes = synth.vqa_state_dict_shapes(cfg)
    get = lambda n: synth.synthetic_tensor(n, shapes[n], seed=4321, device="cuda")      # noqa: E731
    makers = dict(bf16=lambda: VQAWeights(cfg, get, dtype=torch.bfloat16), nf4=lambda: VQAWeights(cfg, get, dtype=torch.float16, quant="nf4"))
    with torch.inference_mode():
        for name in a.dtypes.split(","):
            res[name] = bench_dtype(name, makers[name], vsm, items, missing, conf, a.rounds, min(a.check_items, len(items)))
            print(json.dumps({name: res[name]["median_over_rounds"]}), flush=True)
    res["gpu_after"] = gpu_info()
    print(json.dumps({k: v for k, v in res.items() if k not in a.dtypes.split(",")}))
    if a.out:
        # one run per dtype fits a shorter job: the dtypes of earlier runs already in the file are kept, each with its GPU
        old = json.load(open(a.out)) if os.path.exists(a.out) else {}
        for name in a.dtypes.split(","):
            old[name] = dict(res[name], gpu_before=res["gpu_before"], gpu_after=res["gpu_after"])
        old.update({k: v for k, v in res.items() if k not in ("gpu_before", "gpu_after") and k not in makers})
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(old, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
