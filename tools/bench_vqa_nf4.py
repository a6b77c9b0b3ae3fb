"""SEAL VQA LLM at full size (Vicuna-7B + CLIP-L shapes, random weights) in fp16 and in its 4-bit mode (NF4 Linears, fp16
compute), timed in one process.

The two engines are alternated round by round (fp16, nf4, fp16, ...); every number is the median over the rounds of CUDA-event
times taken after a warm-up (the measures of tools/bench_vqa_dtype.py):
  * prefill of a ~600-token prompt;
  * greedy decode ms/token at B = 1 and B = 8, with the fraction of the HBM roofline computed from the bytes each engine must
    read per step (NF4: half a byte per weight plus an fp32 scale per 64, fp16 lm_head, KV rows) over 3.35 TB/s;
  * one 4-option scoring.
Then the NF4 GEMM alone at the 7B projection shapes: the streaming kernels' share of the HBM roofline at M = 1 and 8, and the
M crossover between the mma.sync streaming kernel and dequant + wgmma tiles (the dispatcher's NF4_SKINNY_MAX_M).
The GPU name, power limit and max SM clock are read in the same run.

    python tools/bench_vqa_nf4.py [--rounds 5] [--steps 32] [--out results.json]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from tools.bench_vqa_dtype import HBM_PEAK, events, gpu_info, make_case
from vstar_b200 import _lib, ops, synth
from vstar_b200.config import VSMConfig
from vstar_b200.vqa import VQAEngine, VQAWeights


def decode_bytes(cfg, B, T, nf4):
    d, inter = cfg.hidden, cfg.intermediate
    n = cfg.n_layers * (4 * d * d + 3 * d * inter)
    weights = (n // 2 + n // 64 * 4 if nf4 else 2 * n) + cfg.vocab * d * 2
    return weights + cfg.n_layers * B * T * 2 * d * 2


def one_round(cfg, eng, c, steps, nf4):
    r = {}
    x = eng.build_embeds(c["q"], c["image"], c["crop"], c["il"], c["ol"])
    T = int(x.shape[0])
    r["prefill_T"] = T
    r["prefill_ms"] = events(lambda: eng.prefill_embeds(eng.build_embeds(c["q"], c["image"], c["crop"], c["il"], c["ol"])))
    ms = events(lambda: [eng.append_tokens([1234], T) for _ in range(steps)]) / steps
    r["decode_B1_ms_per_token"] = ms
    r["decode_B1_hbm_fraction"] = decode_bytes(cfg, 1, T, nf4) / (ms * 1e-3) / HBM_PEAK
    xs = [eng.build_embeds(*q) for q in c["reqs"]]
    _, Tpad, lens = eng.prefill_ragged(xs)
    toks = [1234] * len(lens)
    ms = events(lambda: [eng.decode_ragged(toks, lens, Tpad, 0) for _ in range(steps)]) / steps
    r["decode_B8_ms_per_step"] = ms
    r["decode_B8_hbm_fraction"] = decode_bytes(cfg, len(lens), Tpad, nf4) / (ms * 1e-3) / HBM_PEAK
    r["options4_ms"] = events(lambda: eng.option_losses(c["q"], c["opts"], c["image"], c["crop"], c["il"], c["ol"]))
    return r


def gemm_ms(a, w, force, deq, reps=20):
    _lib.call("vsb_gemm_set_tuning", force, 0)
    try:
        ops.gemm(a, w, deq_scratch=deq)
        return events(lambda: [ops.gemm(a, w, deq_scratch=deq) for _ in range(reps)]) / reps
    finally:
        _lib.call("vsb_gemm_set_tuning", 0, 0)


def gemm_sweep(cfg):
    """per 7B projection shape: streaming kernels' roofline share, and streaming (mma.sync) vs dequant + tile over M"""
    d, inter = cfg.hidden, cfg.intermediate
    shapes = {"qkv": (3 * d, d), "o": (d, d), "gate_up": (2 * inter, d), "down": (d, inter)}
    deq = torch.empty(2 * inter * d, dtype=torch.float16, device="cuda")
    out = {}
    for name, (N, K) in shapes.items():
        w = ops.nf4_quantize((torch.randn(N, K, device="cuda") * K ** -0.5).half())
        row = {}
        for M, force in ((1, 1), (1, 2), (8, 1), (8, 2)):
            a = torch.randn(M, K, device="cuda").half()
            ms = gemm_ms(a, w, force, deq)
            row[f"M{M}_v{force}_ms"] = ms
            row[f"M{M}_v{force}_hbm_fraction"] = (N * K // 2 + N * K // 64 * 4 + 2 * M * (K + N)) / (ms * 1e-3) / HBM_PEAK
        for M in (8, 16, 24, 32, 48, 64):
            a = torch.randn(M, K, device="cuda").half()
            if M <= 32:
                row[f"M{M}_stream_ms"] = gemm_ms(a, w, 2, deq)
            row[f"M{M}_tile_ms"] = min(gemm_ms(a, w, bn, deq) for bn in (64, 128))
        out[name] = row
    cross = {}
    for M in (8, 16, 24, 32):
        s = sum(out[n][f"M{M}_stream_ms"] for n in shapes)
        t = sum(out[n][f"M{M}_tile_ms"] for n in shapes)
        cross[M] = dict(stream_ms=s, tile_ms=t, stream_faster=s < t)
    return out, cross


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=32, help="decode steps per timed window")
    ap.add_argument("--out", default=None, help="also write the result JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vqa_nf4 needs a CUDA GPU (nothing is measured on the CPU)")
    cfg = VSMConfig()
    shapes = synth.vqa_state_dict_shapes(cfg)
    engines, cases, load = {}, {}, {}
    with torch.inference_mode():
        for name, quant in (("fp16", None), ("nf4", "nf4")):
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            w = VQAWeights(cfg, lambda n: synth.synthetic_tensor(n, shapes[n], seed=4321, device="cuda"), dtype=torch.float16, quant=quant)
            load[name] = dict(linear_weight_bytes=w.linear_bytes(), all_bytes=torch.cuda.memory_allocated() - base,
                              load_peak_bytes=torch.cuda.max_memory_allocated() - base)
            engines[name] = VQAEngine(w, max_tokens=1024)
            cases[name] = make_case(cfg, engines[name], torch.float16)
            one_round(cfg, engines[name], cases[name], 4, quant is not None)
        rounds = {k: [] for k in engines}
        for i in range(a.rounds):
            for name in engines:
                rounds[name].append(one_round(cfg, engines[name], cases[name], a.steps, name == "nf4"))
        sweep, cross = gemm_sweep(cfg)
    res = dict(gpu=gpu_info(), rounds=a.rounds, decode_steps=a.steps, hbm_peak_bytes_per_s=HBM_PEAK, weights=load)
    for name, rs in rounds.items():
        res[name] = {k: float(np.median([r[k] for r in rs])) for k in rs[0]}
        res[name + "_spread"] = {k: [float(min(r[k] for r in rs)), float(max(r[k] for r in rs))] for k in rs[0]}
    res["nf4_over_fp16"] = {k: res["nf4"][k] / res["fp16"][k] for k in res["fp16"] if k.endswith("_ms") or "per_" in k}
    res["gemm_nf4"] = sweep
    res["crossover_sum_of_7b_projections"] = cross
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
