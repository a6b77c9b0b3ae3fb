"""Cost of beam search (VQAEngine.beam_search: vsb_beam_candidates_f32 + vsb_copy_cache_rows_b16 per step) next to greedy decoding on
the SEAL VQA LLM at Vicuna-7B + CLIP-L shapes (random weights, bf16), prompt of about 600 rows (340 ids + the 256 image rows).

  * ms per decode step at num_beams k in {1 (the greedy path), 2, 4, 8}, for 64 and 200 new tokens (eos never wins: the ids
    are random and eos = -1), the k values alternated round by round: (time of an N-token call - time of a 1-token call) /
    (N - 1), so the prefill cancels; medians over the rounds;
  * kernel times inside a 32-token beam call from torch.profiler (CUDA activity): the candidate kernel, the row copies and
    the decode attention per step, and their share of the step's GPU time; the attention share at k = 4 against k = 1;
  * the candidate kernel alone on fp32 logits [k, 32000] (CUDA events around `--reps` launches).
The GPU name, power limit and clocks are read in the same run.

    python tools/bench_vqa_beams.py [--rounds 3] [--reps 200] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from tools.bench_vqa_dtype import events
from vstar_b200 import ops, synth
from vstar_b200.config import VSMConfig
from vstar_b200.vqa import VQAEngine, VQAWeights

KS = (1, 2, 4, 8)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
    except (OSError, subprocess.SubprocessError):
        q = ""
    return dict(device=torch.cuda.get_device_name(), nvidia_smi_name_power_clock_maxclock_memclock=q)


def step_times(eng, req, rounds, tokens):
    calls = {k: (lambda N, k=k: eng.generate(*req, max_new_tokens=N, eos_token_id=-1, num_beams=k)) for k in KS}
    for f in calls.values():
        f(3)
    out = {}
    for N in tokens:
        times = {k: [] for k in KS}
        for _ in range(rounds):
            for k, f in calls.items():
                full, one = events(lambda: f(N)), events(lambda: f(1))
                times[k].append((full - one) / (N - 1))
        r = {f"k{k}_ms_per_step": float(np.median(v)) for k, v in times.items()}
        r.update({f"k{k}_ms_per_step_spread": [float(min(v)), float(max(v))] for k, v in times.items()})
        r.update({f"k{k}_over_greedy": r[f"k{k}_ms_per_step"] / r["k1_ms_per_step"] for k in KS})
        out[f"new_tokens_{N}"] = r
    return out


def kernel_shares(eng, req, k, N=32):
    from torch.profiler import ProfilerActivity, profile
    eng.generate(*req, max_new_tokens=N, eos_token_id=-1, num_beams=k)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.generate(*req, max_new_tokens=N, eos_token_id=-1, num_beams=k)
        torch.cuda.synchronize()
    tot = {"candidates": 0.0, "row_copies": 0.0, "attention": 0.0, "all": 0.0}
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if t <= 0:
            continue
        name = e.key.lower()
        tot["all"] += t
        if "beam_candidates" in name:
            tot["candidates"] += t
        elif "copy_cache_rows" in name:
            tot["row_copies"] += t
        elif "attn" in name or "attention" in name:
            tot["attention"] += t
    # the call is one prefill + N - 1 decode steps; per-step numbers divide the beam kernels by N and the decode attention by N - 1
    return dict(candidates_us_per_step=tot["candidates"] / N, row_copies_us_per_step=tot["row_copies"] / max(1, N - 1),
                attention_us_all_call=tot["attention"], gpu_us_all_call=tot["all"],
                candidates_share=tot["candidates"] / tot["all"], row_copies_share=tot["row_copies"] / tot["all"],
                attention_share=tot["attention"] / tot["all"])


def candidate_kernel(rounds, reps):
    out = {}
    for k in KS:
        x = torch.randn(k, 32000, generator=torch.Generator().manual_seed(k)).mul(3).cuda()
        rows = torch.arange(k, dtype=torch.int32, device="cuda").view(1, k)
        sc = -torch.rand(1, k, device="cuda")
        f = lambda: ops.beam_candidates(x, rows, sc, k, torch.bfloat16)
        f()
        t = [events(lambda: [f() for _ in range(reps)]) * 1e3 / reps for _ in range(rounds)]
        out[f"k{k}_us"] = float(np.median(t))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=200, help="kernel launches per timed window")
    ap.add_argument("--out", default=None, help="also write the result JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vqa_beams needs a CUDA GPU (nothing is measured on the CPU)")
    res = dict(gpu_before=gpu_info(), rounds=a.rounds, kernel_reps=a.reps)
    with torch.inference_mode():
        res["candidate_kernel_V32000_bf16"] = candidate_kernel(a.rounds, a.reps)
        cfg = VSMConfig()
        shapes = synth.vqa_state_dict_shapes(cfg)
        w = VQAWeights(cfg, lambda n: synth.synthetic_tensor(n, shapes[n], seed=4321, device="cuda"), dtype=torch.bfloat16)
        eng = VQAEngine(w, max_tokens=1024)
        rng = np.random.default_rng(0)
        image = torch.randn(1, 3, 224, 224, generator=torch.Generator().manual_seed(0)).to(torch.bfloat16).cuda()
        ids = [1] + rng.integers(1000, 30000, 200).tolist() + [-200] + rng.integers(1000, 30000, 140).tolist()
        req = (ids, image, None, [True], None)
        res["prompt_rows"] = int(eng.build_embeds(*req).shape[0])
        res["decode_7b_bf16"] = step_times(eng, req, a.rounds, (64, 200))
        res["profile_32_tokens"] = {f"k{k}": kernel_shares(eng, req, k) for k in KS}
        p = res["profile_32_tokens"]
        res["attention_share_k4_over_k1"] = p["k4"]["attention_share"] / p["k1"]["attention_share"]
    res["gpu_after"] = gpu_info()
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
