"""What the paged KV cache (DecodeStream(kv_pages=N)) costs and what it buys, on the SEAL VQA LLM at Vicuna-7B + CLIP-L shapes
with random weights, in bf16 and NF4, on the 64-request workload of tools/bench_vqa_stream.py (300-900 prompt rows, 8-512
answer tokens; random weights never emit eos, so every request runs to its own max_new_tokens).

  * equal slots: a contiguous and a paged stream of 16 slots at 1536 positions, the paged pool large enough never to refuse a
    request, so both run the same schedule: ms per decode step, tokens/s, whether the tokens agree.  The cost of the page
    indirection.  torch.profiler, in a run of its own: the paged attention kernel's time per step against the contiguous one's.
  * equal KV bytes: the cache of 16 and of 32 contiguous slots at 1536 positions (1.125 GiB per slot in bf16), against a paged
    pool of the same bytes with max_slots raised to every request (greedy) or every request's beams (num_beams = 4).  A request is
    admitted when its slots and the pages it reserves are free.  Tokens/s, mean requests running per decode step, peak device
    memory of the run.
The two arms of each comparison alternate, `rounds` times; medians and [min, max] spreads.  The GPU name, power limit and
clocks are read in the same run.

    python tools/bench_vqa_stream_paged.py [--requests 64] [--rounds 2] [--dtypes bf16,nf4] [--out results.json]
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
from vstar_b200 import synth
from vstar_b200.config import VSMConfig
from vstar_b200.kv_pages import PAGE_ROWS
from vstar_b200.vqa import VQAEngine, VQAWeights

POSITIONS = 1536                                   # the engine default: rows of one contiguous slot
BEAMS = 4


def equal_bytes_pages(slots, positions=POSITIONS):
    """pages of PAGE_ROWS k|v rows (2d) in the bytes of `slots` contiguous slots of `positions` q|k|v rows (3d)"""
    return slots * positions * 3 // (PAGE_ROWS * 2)


def run(eng, reqs, lens, max_slots, kv_pages=None, num_beams=1):
    """every request through one stream, admitted in order as its slots (and pages) free -> (tokens, stats)"""
    kw = {} if num_beams == 1 else dict(num_beams=num_beams)
    T = [eng.spliced_length(r[0], 0, r[3]) for r in reqs]
    outs = [None] * len(reqs)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    m0 = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    st = eng.decode_stream(max_slots, max_positions=POSITIONS, eos_token_id=-1, kv_pages=kv_pages)
    owner, nxt, t_step, running = {}, 0, 0.0, 0

    def fits():
        if st.free_slots < num_beams:
            return False
        return st.pages is None or st.pages.need(T[nxt], lens[nxt], num_beams) <= st.pages.free_pages

    def admit():
        nonlocal nxt
        while nxt < len(reqs) and fits():
            owner[st.admit(reqs[nxt], lens[nxt], **kw).id] = nxt
            nxt += 1
    admit()
    remaining = len(reqs)
    while remaining:
        running += len(st.active)
        t1 = time.perf_counter()
        done = st.step()                                      # ends in the device-to-host copy of the step's tokens
        t_step += time.perf_counter() - t1
        for r, toks in done:
            outs[owner[r.id]] = list(toks)
            remaining -= 1
        admit()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    res = dict(wall_s=wall, steps=st.steps, decode_s=t_step, requests_per_step=running / max(1, st.steps),
               peak_stream_gib=(torch.cuda.max_memory_allocated() - m0) / 2 ** 30,
               kv_gib=st._cache.numel() * st._cache.element_size() / 2 ** 30)
    st.close()
    torch.cuda.empty_cache()
    return outs, res


def summarise(runs, tokens):
    wall = [r["wall_s"] for r in runs]
    step = [1e3 * r["decode_s"] / max(1, r["steps"]) for r in runs]
    return dict(wall_s=float(np.median(wall)), wall_s_spread=[min(wall), max(wall)], tokens_per_s=tokens / float(np.median(wall)),
                tokens_per_s_spread=[tokens / max(wall), tokens / min(wall)], ms_per_decode_step=float(np.median(step)),
                ms_per_decode_step_spread=[min(step), max(step)], decode_steps=runs[0]["steps"],
                mean_requests_per_step=runs[0]["requests_per_step"], peak_stream_gib=max(r["peak_stream_gib"] for r in runs),
                kv_gib=runs[0]["kv_gib"])


def compare(eng, reqs, lens, rounds, arms, tokens):
    """arms: {name: run() keywords}, alternated `rounds` times -> {name: summary} and whether every arm gave the same tokens"""
    res = {n: [] for n in arms}
    outs = {}
    for _ in range(rounds):
        for n, kw in arms.items():
            outs[n], r = run(eng, reqs, lens, **kw)
            res[n].append(r)
    first = next(iter(outs.values()))
    return {n: summarise(v, tokens) for n, v in res.items()}, all(o == first for o in outs.values())


def attention_time(eng, reqs, slots=16, steps=32, kv_pages=None):
    """torch.profiler over `steps` stream steps of `slots` requests: device time per step of the slot-attention kernel"""
    from torch.profiler import ProfilerActivity, profile
    st = eng.decode_stream(slots, max_positions=POSITIONS, eos_token_id=-1, kv_pages=kv_pages)
    for r in reqs[:slots]:
        st.admit(r, steps + 2)
    st.step()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            st.step()
        torch.cuda.synchronize()
    st.close()
    att = tot = 0.0
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if t <= 0:
            continue
        tot += t
        if "attn_decode_slots_kernel" in e.key or "attn_decode_paged_kernel" in e.key:
            att += t
    return dict(attention_us_per_step=att / steps, gpu_us_per_step=tot / steps)


def bench_dtype(make_weights, n, rounds):
    eng = VQAEngine(make_weights(), max_tokens=POSITIONS)
    reqs, lens = workload(n)
    reqs = [(ids, img.to(eng.dtype).cuda(), c, il, ol) for ids, img, c, il, ol in reqs]
    tokens = sum(lens)
    out = dict(requests=n, generated_tokens=tokens, page_rows=PAGE_ROWS, positions=POSITIONS)
    ample = 16 * -(-POSITIONS // PAGE_ROWS)                     # every slot's full row count: the pool never refuses
    run(eng, reqs[:4], [4] * 4, 4)                              # warm-up of every kernel family of both arms
    run(eng, reqs[:4], [4] * 4, 4, kv_pages=ample)
    run(eng, reqs[:2], [4] * 2, 8, num_beams=BEAMS)
    run(eng, reqs[:2], [4] * 2, 8, kv_pages=ample, num_beams=BEAMS)
    s, same = compare(eng, reqs, lens, rounds, dict(contiguous=dict(max_slots=16), paged=dict(max_slots=16, kv_pages=ample)), tokens)
    out["equal_slots_16"] = dict(s, same_tokens=same)
    out["equal_slots_16"]["attention"] = dict(contiguous=attention_time(eng, reqs), paged=attention_time(eng, reqs, kv_pages=ample))
    for budget in (16, 32):
        pages = equal_bytes_pages(budget)
        for k in (1, BEAMS):
            arms = dict(contiguous=dict(max_slots=budget, num_beams=k), paged=dict(max_slots=n * k, kv_pages=pages, num_beams=k))
            s, same = compare(eng, reqs, lens, rounds, arms, tokens)
            out[f"equal_bytes_{budget}_{'greedy' if k == 1 else f'beam{k}'}"] = dict(s, kv_pages=pages, same_tokens=same)
    del eng
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--dtypes", default="bf16,nf4")
    ap.add_argument("--out", default=None, help="also write the result JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vqa_stream_paged needs a CUDA GPU (nothing is measured on the CPU)")
    res = dict(gpu_before=gpu_info(), rounds=a.rounds)
    cfg = VSMConfig()
    shapes = synth.vqa_state_dict_shapes(cfg)
    get = lambda n: synth.synthetic_tensor(n, shapes[n], seed=4321, device="cuda")
    makers = dict(bf16=lambda: VQAWeights(cfg, get, dtype=torch.bfloat16),
                  nf4=lambda: VQAWeights(cfg, get, dtype=torch.float16, quant="nf4"))
    with torch.inference_mode():
        for name in a.dtypes.split(","):
            res[name] = bench_dtype(makers[name], a.requests, a.rounds)
            print(json.dumps({name: res[name]}, indent=1), flush=True)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
