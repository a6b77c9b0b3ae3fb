"""What iteration-level admission (VQAEngine.decode_stream) gains over the static batch of generate_batch, on the SEAL VQA LLM at
Vicuna-7B + CLIP-L shapes with random weights, in bf16 and in NF4 (load_4bit).

Workload: N requests with SEAL-shaped prompts (text ids + the 256 image rows: 300-900 rows) and answer lengths drawn once from
a seeded log-uniform distribution over 8-512 tokens.  Random weights never emit eos, so every request runs to its own
max_new_tokens.  For B = 8, 16 and 32:
  * static: generate_batch over consecutive chunks of B requests, each with its own max_new_tokens (a chunk steps until its
    longest answer ends; finished rows idle);
  * stream: one decode stream with B slots, the next request admitted whenever a slot frees.
Reported per (dtype, B, mode): wall time, generated tokens/s, mean occupied slots per decode step (rows still generating),
ms per decode step (decode time without the CLIP + prefill work); medians over rounds that alternate the two modes.
torch.profiler, in a run of its own: the slot-decode attention's share of the GPU time of 32 stream steps at B = 16.
The GPU name, power limit and clocks are read in the same run.

    python tools/bench_vqa_stream.py [--requests 64] [--rounds 3] [--out results.json]
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
from vstar_b200 import synth
from vstar_b200.config import VSMConfig
from vstar_b200.vqa import VQAEngine, VQAWeights

BS = (8, 16, 32)


def workload(n, seed=0):
    """-> requests (ids, image, None, [True], None) and their max_new_tokens"""
    rng = np.random.default_rng(seed)
    gen = torch.Generator().manual_seed(seed)
    reqs, lens = [], []
    for _ in range(n):
        text = int(rng.integers(44, 645))                      # + 256 image rows = 300-900 prompt rows
        pre = int(rng.integers(30, 40))
        ids = [1] + rng.integers(1000, 30000, pre).tolist() + [-200] + rng.integers(1000, 30000, text - pre - 1).tolist()
        reqs.append((ids, torch.randn(1, 3, 224, 224, generator=gen), None, [True], None))
        lens.append(int(round(float(np.exp(rng.uniform(np.log(8), np.log(512)))))))
    return reqs, lens


class Timer:
    """synchronised host time spent inside the wrapped engine methods (the CLIP + prefill work of a call)"""

    def __init__(self, eng, names):
        self.t = 0.0
        for name in names:
            f = getattr(eng, name)

            def wrapped(*a, _f=f, **k):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                r = _f(*a, **k)
                torch.cuda.synchronize()
                self.t += time.perf_counter() - t0
                return r
            setattr(eng, name, wrapped)
        self.eng, self.names = eng, names

    def remove(self):
        for name in self.names:
            delattr(self.eng, name)


def free_engine_cache(eng):
    eng._cache = None
    eng._cache_shape = None
    torch.cuda.empty_cache()


def run_static(eng, reqs, lens, B):
    outs = []
    steps = 0
    tm = Timer(eng, ["build_embeds_batch", "prefill_ragged"])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(0, len(reqs), B):
        chunk, budgets = reqs[i:i + B], lens[i:i + B]
        # generate_batch takes one max_new_tokens per call: the chunk runs to its longest budget, each answer is cut to its own
        o = eng.generate_batch(chunk, max_new_tokens=max(budgets), eos_token_id=-1)
        outs += [x[:n] for x, n in zip(o, budgets)]
        steps += max(budgets) - 1
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    tm.remove()
    free_engine_cache(eng)
    return outs, dict(wall_s=wall, steps=steps, decode_s=wall - tm.t)


def run_stream(eng, reqs, lens, B):
    outs = [None] * len(reqs)
    longest = max(eng.spliced_length(r[0], 0, r[3]) + n for r, n in zip(reqs, lens))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    st = eng.decode_stream(B, max_positions=longest, eos_token_id=-1)
    owner, nxt, t_step = {}, 0, 0.0
    while nxt < len(reqs) and st.free_slots:
        owner[st.admit(reqs[nxt], lens[nxt]).id] = nxt
        nxt += 1
    remaining = len(reqs)
    while remaining:
        t1 = time.perf_counter()
        done = st.step()                                      # ends in the device-to-host copy of the step's tokens
        t_step += time.perf_counter() - t1
        for r, toks in done:
            outs[owner[r.id]] = toks
            remaining -= 1
        while nxt < len(reqs) and st.free_slots:
            owner[st.admit(reqs[nxt], lens[nxt]).id] = nxt
            nxt += 1
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    res = dict(wall_s=wall, steps=st.steps, decode_s=t_step, occupied=st.occupied)
    st.close()
    return outs, res


def summarise(runs, total_tokens, B, lens):
    wall = float(np.median([r["wall_s"] for r in runs]))
    dec = float(np.median([r["decode_s"] / max(1, r["steps"]) for r in runs]))
    r0 = runs[0]
    occ = r0["occupied"] / r0["steps"] if "occupied" in r0 else (total_tokens - len(lens)) / r0["steps"]
    return dict(wall_s=wall, wall_s_spread=[float(min(r["wall_s"] for r in runs)), float(max(r["wall_s"] for r in runs))],
                tokens_per_s=total_tokens / wall, mean_occupied_slots=occ, slots=B, ms_per_decode_step=1e3 * dec, decode_steps=r0["steps"])


def attention_share(eng, reqs, B=16, steps=32):
    from torch.profiler import ProfilerActivity, profile
    st = eng.decode_stream(B, max_positions=1024, eos_token_id=-1)
    for r in reqs[:B]:
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
        if "attn_decode_slots" in e.key:
            att += t
    return dict(slots=B, steps=steps, attention_us_per_step=att / steps, gpu_us_per_step=tot / steps, attention_share=att / tot)


def bench_dtype(name, make_weights, n, rounds):
    eng = VQAEngine(make_weights(), max_tokens=1024)
    reqs, lens = workload(n)
    reqs = [(ids, img.to(eng.dtype).cuda(), c, il, ol) for ids, img, c, il, ol in reqs]
    total = sum(lens)
    out = dict(requests=n, generated_tokens=total, prompt_rows=[int(eng.spliced_length(r[0], 0, r[3])) for r in reqs], answer_tokens=lens)
    run_static(eng, reqs[:4], [4] * 4, 4)                     # warm-up: every kernel family of both modes
    run_stream(eng, reqs[:4], [4] * 4, 4)
    for B in BS:
        st_runs, sm_runs = [], []
        for _ in range(rounds):
            o_static, r = run_static(eng, reqs, lens, B)
            st_runs.append(r)
            o_stream, r = run_stream(eng, reqs, lens, B)
            sm_runs.append(r)
        s, m = summarise(st_runs, total, B, lens), summarise(sm_runs, total, B, lens)
        out[f"B{B}"] = dict(static=s, stream=m, stream_speedup_wall=s["wall_s"] / m["wall_s"],
                            same_tokens=sum(a == b for a, b in zip(o_static, o_stream)) / n)
    out["profile"] = attention_share(eng, reqs)
    del eng
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--dtypes", default="bf16,nf4")
    ap.add_argument("--out", default=None, help="also write the result JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vqa_stream needs a CUDA GPU (nothing is measured on the CPU)")
    res = dict(gpu_before=gpu_info(), rounds=a.rounds)
    cfg = VSMConfig()
    shapes = synth.vqa_state_dict_shapes(cfg)
    get = lambda n: synth.synthetic_tensor(n, shapes[n], seed=4321, device="cuda")
    makers = dict(bf16=lambda: VQAWeights(cfg, get, dtype=torch.bfloat16),
                  nf4=lambda: VQAWeights(cfg, get, dtype=torch.float16, quant="nf4"))
    with torch.inference_mode():
        for name in a.dtypes.split(","):
            res[name] = bench_dtype(name, makers[name], a.requests, a.rounds)
            print(json.dumps({name: {k: v for k, v in res[name].items() if k.startswith("B") or k == "profile"}}, indent=1), flush=True)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
