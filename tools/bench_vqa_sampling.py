"""Cost of sampled decoding (vsb_sample_rows_f32) next to greedy decoding (vsb_argmax_rows_f32) on the SEAL VQA LLM.

  * kernel time of argmax_rows and of the sampler on fp32 logits [B, 32000] (B = 1, 8, 32, 64), for top_k = 50 and for
    top_k = 0, top_p = 0.9 (nucleus over the whole vocabulary, the binary-search path), T = 0.7, bf16 rounding: CUDA events
    around `--reps` launches, the kernels alternated round by round, medians over the rounds;
  * decode ms/token at Vicuna-7B + CLIP-L shapes (random weights, bf16): greedy generate / generate_batch against sampled
    (T = 0.7, top_k = 50, top_p = 0.9) at B = 1 and B = 8, alternated round by round.  ms/token = (time of a
    `--tokens`-token call - time of a 1-token call) / (tokens - 1), so the prefill cancels; medians over the rounds.
The GPU name, power limit and max SM clock are read in the same run.

    python tools/bench_vqa_sampling.py [--rounds 5] [--tokens 33] [--reps 200] [--out results.json]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from tools.bench_vqa_dtype import events, gpu_info, make_case
from vstar_b200 import ops, synth
from vstar_b200.config import VSMConfig
from vstar_b200.vqa import VQAEngine, VQAWeights

SAMPLED = dict(temperature=0.7, top_k=50, top_p=0.9)


def kernel_times(rounds, reps):
    n = 32000
    out = {}
    for B in (1, 8, 32, 64):
        x = torch.randn(B, n, generator=torch.Generator().manual_seed(B)).mul(2.5).cuda()
        seeds = torch.arange(B, dtype=torch.int64, device="cuda") * 7919 + 1
        fns = {"argmax": lambda: ops.argmax_rows(x),
               "sample_top_k50": lambda: ops.sample_rows(x, 0.7, 50, None, torch.bfloat16, seeds, 3),
               "sample_top_k0_top_p0.9": lambda: ops.sample_rows(x, 0.7, 0, 0.9, torch.bfloat16, seeds, 3)}
        for f in fns.values():
            f()
        times = {k: [] for k in fns}
        for _ in range(rounds):
            for k, f in fns.items():
                times[k].append(events(lambda: [f() for _ in range(reps)]) * 1e3 / reps)
        out[f"B{B}"] = {k + "_us": float(np.median(v)) for k, v in times.items()}
        out[f"B{B}"].update({k + "_us_spread": [float(min(v)), float(max(v))] for k, v in times.items()})
    return out


def decode_times(eng, c, rounds, tokens):
    req = (c["q"], c["image"], c["crop"], c["il"], c["ol"])
    reqs = c["reqs"]
    calls = {
        "B1_greedy": lambda N: eng.generate(*req, max_new_tokens=N, eos_token_id=-1),
        "B1_sampled": lambda N: eng.generate(*req, max_new_tokens=N, eos_token_id=-1, seed=5, **SAMPLED),
        "B8_greedy": lambda N: eng.generate_batch(reqs, max_new_tokens=N, eos_token_id=-1),
        "B8_sampled": lambda N: eng.generate_batch(reqs, max_new_tokens=N, eos_token_id=-1, seeds=list(range(8)), **SAMPLED),
    }
    for f in calls.values():                                       # warm-up of every shape
        f(2)
    times = {k: [] for k in calls}
    for _ in range(rounds):
        for k, f in calls.items():
            full, one = events(lambda: f(tokens)), events(lambda: f(1))
            times[k].append((full - one) / (tokens - 1))
    res = {k + "_ms_per_token": float(np.median(v)) for k, v in times.items()}
    res.update({k + "_ms_per_token_spread": [float(min(v)), float(max(v))] for k, v in times.items()})
    for B in ("B1", "B8"):
        res[B + "_sampled_over_greedy"] = res[B + "_sampled_ms_per_token"] / res[B + "_greedy_ms_per_token"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--tokens", type=int, default=33, help="new tokens of the long generate call")
    ap.add_argument("--reps", type=int, default=200, help="kernel launches per timed window")
    ap.add_argument("--out", default=None, help="also write the result JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vqa_sampling needs a CUDA GPU (nothing is measured on the CPU)")
    res = dict(gpu=gpu_info(), rounds=a.rounds, tokens=a.tokens, kernel_reps=a.reps, sampled=SAMPLED)
    with torch.inference_mode():
        res["kernel_n32000"] = kernel_times(a.rounds, a.reps)
        cfg = VSMConfig()
        shapes = synth.vqa_state_dict_shapes(cfg)
        w = VQAWeights(cfg, lambda n: synth.synthetic_tensor(n, shapes[n], seed=4321, device="cuda"), dtype=torch.bfloat16)
        eng = VQAEngine(w, max_tokens=1024)
        res["decode_7b_bf16"] = decode_times(eng, make_case(cfg, eng, torch.bfloat16), a.rounds, a.tokens)
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
