"""What growing the paged decode stream's pages on demand, with preemption by swap (DecodeStream(kv_pages=N, kv_swap_pages=M)),
buys over reserving every request's pages at admission (kv_pages=N alone), on the SEAL VQA LLM at Vicuna-7B + CLIP-L shapes with
random weights, in bf16 and NF4.

Workload: the 64 requests of tools/bench_vqa_stream.py (300-900 prompt rows, answer lengths drawn in 8-512), every one admitted
with max_new_tokens = 512 as the SEAL loop admits its answers.  Random weights never emit eos, so request i is ended after its
drawn length by a DecodeStream subclass (EndsAt) that stands in for a trained model's eos; both arms use it the same way.  The
reserve-ahead arm therefore reserves ceil((T + 512) / 64) pages per row, while the growing arm takes the pages rows are written.

  * equal KV bytes: pools of the bytes of 16 and of 32 contiguous slots at 1536 positions, greedy and beam k = 4; the growing
    arm gets a pinned host swap area of --swap-pages pages.  Wall time, tokens/s, mean requests decoding per step,
    preemptions and bytes swapped each way, peak device memory.  The arms alternate --rounds times.
  * forced preemption: a greedy run on a pool of twice the largest request, small enough to preempt often; and the swap
    kernel's GB/s in each direction over 64 pages against a cudaMemcpyAsync (torch copy_) of the same bytes between the same
    pinned buffer and the device, CUDA events around 10 repetitions each.
The GPU name, power limit and clocks are read in the same run.

    python tools/bench_vqa_stream_swap.py [--requests 64] [--rounds 1] [--dtypes bf16,nf4] [--swap-pages 1152] [--out results.json]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from tools.bench_vqa_beams import gpu_info
from tools.bench_vqa_stream import workload
from tools.bench_vqa_stream_paged import POSITIONS, equal_bytes_pages
from vstar_b200 import ops, synth
from vstar_b200.config import VSMConfig
from vstar_b200.kv_pages import PAGE_ROWS
from vstar_b200.vqa import DecodeStream, VQAEngine, VQAWeights

BUDGET = 512                                       # seal.OPEN_MAX_NEW_TOKENS
BEAMS = 4


class EndsAt(DecodeStream):
    """request i (in admission order) ends after ends[i] tokens: a trained model's eos, which random weights never emit"""

    def __init__(self, *a, ends, **kw):
        super().__init__(*a, **kw)
        self.ends = ends

    def _ended(self, r):
        return len(r.tokens) >= self.ends[r.id] or super()._ended(r)

    def _beam_advance(self, r, cand):
        q = super()._beam_advance(r, cand)
        if q is not None and len(r.beam.beams[0]) >= self.ends[r.id]:
            r.tokens, r.score = r.beam.finalize()
            return None
        return q


def _free_host_cache():
    if hasattr(torch._C, "_host_emptyCache"):
        torch._C._host_emptyCache()


def run(eng, reqs, ends, max_slots, kv_pages, kv_swap_pages=None, num_beams=1):
    """every request through one stream with max_new_tokens = BUDGET, admitted in order when the pool's rule allows"""
    kw = {} if num_beams == 1 else dict(num_beams=num_beams)
    T = [eng.spliced_length(r[0], 0, r[3]) for r in reqs]
    outs = [None] * len(reqs)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    m0 = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    st = EndsAt(eng, max_slots, POSITIONS, -1, kv_pages=kv_pages, kv_swap_pages=kv_swap_pages, ends=ends)
    owner, nxt, running = {}, 0, 0

    def fits():
        rows = st.free_rows(num_beams)
        if rows is None:
            return False
        if st.growing:
            return st.pages.can_admit(rows, T[nxt], BUDGET)
        return st.pages.need(T[nxt], BUDGET, num_beams) <= st.pages.free_pages

    def admit():
        nonlocal nxt
        while nxt < len(reqs) and fits():
            owner[st.admit(reqs[nxt], BUDGET, **kw).id] = nxt
            nxt += 1
    admit()
    remaining = len(reqs)
    while remaining:
        running += len(st.active)
        for r, toks in st.step():
            outs[owner[r.id]] = list(toks)
            remaining -= 1
        admit()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    page_bytes = st._cache[:, 0].numel() * st._cache.element_size()
    res = dict(wall_s=wall, steps=st.steps, requests_per_step=running / max(1, st.steps),
               peak_stream_gib=(torch.cuda.max_memory_allocated() - m0) / 2 ** 30, preemptions=st.preemptions,
               swapped_out_gib=st.swapped_pages * page_bytes / 2 ** 30, swapped_in_gib=st.restored_pages * page_bytes / 2 ** 30)
    st.close()
    del st
    torch.cuda.empty_cache()
    return outs, res


def summarise(runs, tokens):
    wall = [r["wall_s"] for r in runs]
    keep = ("steps", "requests_per_step", "preemptions", "swapped_out_gib", "swapped_in_gib")
    return dict(wall_s=float(np.median(wall)), wall_s_spread=[min(wall), max(wall)], tokens_per_s=tokens / float(np.median(wall)),
                **{k: runs[0][k] for k in keep}, peak_stream_gib=max(r["peak_stream_gib"] for r in runs))


def compare(eng, reqs, ends, rounds, arms, tokens):
    res = {n: [] for n in arms}
    outs = {}
    for _ in range(rounds):
        for n, kw in arms.items():
            outs[n], r = run(eng, reqs, ends, **kw)
            res[n].append(r)
    first = next(iter(outs.values()))
    return {n: summarise(v, tokens) for n, v in res.items()}, all(o == first for o in outs.values())


def swap_rate(eng, n_pages=64, reps=10):
    """GB/s of vsb_swap_pages_b16 out and in over n_pages pages, and of torch copy_ (cudaMemcpyAsync) of the same bytes"""
    c = eng.cfg
    pool = torch.randn((c.n_layers, n_pages, PAGE_ROWS, 2 * c.hidden), device="cuda").to(eng.dtype)
    host = torch.empty((n_pages, c.n_layers, PAGE_ROWS, 2 * c.hidden), dtype=eng.dtype, pin_memory=True)
    flat_dev = torch.empty(host.shape, dtype=eng.dtype, device="cuda")
    pairs = list(zip(range(n_pages), range(n_pages)))
    nbytes = pool.numel() * pool.element_size()
    calls = dict(kernel_to_host=lambda: ops.swap_pages(pool, host, pairs, True), kernel_to_device=lambda: ops.swap_pages(pool, host, pairs, False),
                 memcpy_to_host=lambda: host.copy_(flat_dev, non_blocking=True), memcpy_to_device=lambda: flat_dev.copy_(host, non_blocking=True))
    out = dict(bytes=nbytes)
    for name, f in calls.items():
        f()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            f()
        b.record()
        b.synchronize()
        out[name + "_gb_s"] = reps * nbytes / (a.elapsed_time(b) * 1e-3) / 1e9
    ops.swap_pages(pool, host, pairs, True)
    back = torch.empty_like(pool)
    ops.swap_pages(back, host, pairs, False)
    torch.cuda.synchronize()
    out["round_trip_bit_identical"] = bool(torch.equal(back.view(torch.int16), pool.view(torch.int16)))
    del pool, host, flat_dev, back
    torch.cuda.empty_cache()
    _free_host_cache()
    return out


def bench_dtype(make_weights, n, rounds, swap_pages):
    eng = VQAEngine(make_weights(), max_tokens=POSITIONS)
    reqs, ends = workload(n)
    reqs = [(ids, img.to(eng.dtype).cuda(), c, il, ol) for ids, img, c, il, ol in reqs]
    tokens = sum(ends)
    out = dict(requests=n, generated_tokens=tokens, max_new_tokens=BUDGET, page_rows=PAGE_ROWS, positions=POSITIONS, swap_pages=swap_pages)
    page = eng.cfg.n_layers * PAGE_ROWS * 2 * eng.cfg.hidden * 2
    out["swap_area_gib"] = swap_pages * page / 2 ** 30
    ample = 16 * -(-POSITIONS // PAGE_ROWS)
    run(eng, reqs[:4], [4] * 4, 4, ample)                                    # warm-up of every kernel family of both arms
    run(eng, reqs[:4], [4] * 4, 4, ample, swap_pages)
    run(eng, reqs[:2], [4] * 2, 8, ample, num_beams=BEAMS)
    run(eng, reqs[:2], [4] * 2, 8, ample, swap_pages, num_beams=BEAMS)
    for slots in (16, 32):
        pages = equal_bytes_pages(slots)
        for k in (1, BEAMS):
            arms = dict(reserve=dict(max_slots=n * k, kv_pages=pages, num_beams=k),
                        grow_swap=dict(max_slots=n * k, kv_pages=pages, kv_swap_pages=swap_pages, num_beams=k))
            s, same = compare(eng, reqs, ends, rounds, arms, tokens)
            out[f"equal_bytes_{slots}_{'greedy' if k == 1 else f'beam{k}'}"] = dict(s, kv_pages=pages, same_tokens=same)
            print(json.dumps({f"{slots}/{k}": s}), flush=True)
    T = [eng.spliced_length(r[0], 0, r[3]) for r in reqs]
    small = 2 * max(-(-(t + BUDGET) // PAGE_ROWS) for t in T)
    s, same = compare(eng, reqs[:24], ends[:24], 1, dict(reserve=dict(max_slots=24, kv_pages=small),
                                                        grow_swap=dict(max_slots=24, kv_pages=small, kv_swap_pages=swap_pages)),
                      sum(ends[:24]))
    out["forced_preemption_greedy_24"] = dict(s, kv_pages=small, same_tokens=same, swap_rate=swap_rate(eng))
    del eng
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--dtypes", default="bf16,nf4")
    ap.add_argument("--swap-pages", type=int, default=2 * equal_bytes_pages(16), help="pinned host swap area of the growing arm, in pages")
    ap.add_argument("--out", default=None, help="also write the result JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vqa_stream_swap needs a CUDA GPU (nothing is measured on the CPU)")
    res = dict(gpu_before=gpu_info(), rounds=a.rounds)
    cfg = VSMConfig()
    shapes = synth.vqa_state_dict_shapes(cfg)
    get = lambda n: synth.synthetic_tensor(n, shapes[n], seed=4321, device="cuda")
    makers = dict(bf16=lambda: VQAWeights(cfg, get, dtype=torch.bfloat16),
                  nf4=lambda: VQAWeights(cfg, get, dtype=torch.float16, quant="nf4"))
    with torch.inference_mode():
        for name in a.dtypes.split(","):
            res[name] = bench_dtype(makers[name], a.requests, a.rounds, a.swap_pages)
            print(json.dumps({name: res[name]}, indent=1), flush=True)
            _free_host_cache()
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
