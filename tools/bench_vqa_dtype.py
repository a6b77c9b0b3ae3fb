"""SEAL VQA LLM at full size (Vicuna-7B + CLIP-L shapes, random weights) in bf16 and in fp16, timed in one process.

The two engines are alternated round by round (bf16, fp16, bf16, ...) so that clock and neighbour noise hits both alike; every
number is the median over the rounds of CUDA-event times taken after a warm-up:
  * prefill of a ~600-token prompt (image and one object crop as 256 CLIP rows each, ~90 text tokens);
  * greedy decode ms/token at B = 1 (append_tokens) and B = 8 (decode_ragged after prefill_ragged), with the fraction of the HBM
    roofline: (weight bytes + KV-cache bytes read per step) / time / 3.35 TB/s (H100 SXM data sheet);
  * one 4-option scoring (option_losses, every option in one pass).
The GPU name, power limit and max SM clock are read in the same run and printed beside the numbers.

    python tools/bench_vqa_dtype.py [--rounds 5] [--steps 32] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from vstar_b200 import synth
from vstar_b200.config import VSMConfig
from vstar_b200.vqa import VQAEngine, VQAWeights

HBM_PEAK = 3.35e12          # bytes/s, H100 SXM data sheet


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().split("\n")[0]
    except (OSError, subprocess.SubprocessError):
        q = ""
    return dict(device=torch.cuda.get_device_name(), nvidia_smi=q)


def events(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def decode_bytes(cfg, B, T):
    """bytes one decode step must read: every weight of the 32 layers and lm_head once, plus B sequences' K/V rows"""
    d, inter = cfg.hidden, cfg.intermediate
    weights = cfg.n_layers * (4 * d * d + 3 * d * inter) * 2 + cfg.vocab * d * 2
    return weights + cfg.n_layers * B * T * 2 * d * 2


def make_case(cfg, eng, dtype):
    gen = torch.Generator().manual_seed(0)
    image = torch.randn(1, 3, 224, 224, generator=gen).to(dtype).cuda()
    crop = torch.randn(1, 3, 224, 224, generator=gen).to(dtype).cuda()
    rng = np.random.default_rng(0)
    q = [1] + rng.integers(1000, 30000, 40).tolist() + [-200] + rng.integers(1000, 30000, 30).tolist() + [-300] + \
        rng.integers(1000, 30000, 18).tolist()
    opts = [rng.integers(1000, 30000, 6).tolist() for _ in range(4)]
    reqs = [([1] + rng.integers(1000, 30000, 30 + 3 * i).tolist() + [-200] + rng.integers(1000, 30000, 20 + 5 * i).tolist(), image, None,
             [True], None) for i in range(8)]
    return dict(q=q, image=image, crop=crop, il=[True], ol=[True], opts=opts, reqs=reqs)


def one_round(cfg, eng, c, steps):
    r = {}
    x = eng.build_embeds(c["q"], c["image"], c["crop"], c["il"], c["ol"])
    T = int(x.shape[0])
    r["prefill_T"] = T
    r["prefill_ms"] = events(lambda: eng.prefill_embeds(eng.build_embeds(c["q"], c["image"], c["crop"], c["il"], c["ol"])))
    tok = [1234]
    ms = events(lambda: [eng.append_tokens(tok, T) for _ in range(steps)]) / steps
    r["decode_B1_ms_per_token"] = ms
    r["decode_B1_hbm_fraction"] = decode_bytes(cfg, 1, T) / (ms * 1e-3) / HBM_PEAK
    xs = [eng.build_embeds(*q) for q in c["reqs"]]
    _, Tpad, lens = eng.prefill_ragged(xs)
    toks = [1234] * len(lens)
    ms = events(lambda: [eng.decode_ragged(toks, lens, Tpad, 0) for _ in range(steps)]) / steps
    r["decode_B8_ms_per_step"] = ms
    r["decode_B8_hbm_fraction"] = decode_bytes(cfg, len(lens), Tpad) / (ms * 1e-3) / HBM_PEAK
    r["options4_ms"] = events(lambda: eng.option_losses(c["q"], c["opts"], c["image"], c["crop"], c["il"], c["ol"]))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=32, help="decode steps per timed window")
    ap.add_argument("--out", default=None, help="also write the result JSON here")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vqa_dtype needs a CUDA GPU (nothing is measured on the CPU)")
    cfg = VSMConfig()
    shapes = synth.vqa_state_dict_shapes(cfg)
    engines, cases = {}, {}
    with torch.inference_mode():
        for name, dt in (("bf16", torch.bfloat16), ("fp16", torch.float16)):
            w = VQAWeights(cfg, lambda n: synth.synthetic_tensor(n, shapes[n], seed=4321, device="cuda"), dtype=dt)
            engines[name] = VQAEngine(w, max_tokens=1024)
            cases[name] = make_case(cfg, engines[name], dt)
            one_round(cfg, engines[name], cases[name], 4)                 # warm-up: kernel attributes, tensor maps, cache sizes
        rounds = {k: [] for k in engines}
        for i in range(a.rounds):
            for name in engines:
                rounds[name].append(one_round(cfg, engines[name], cases[name], a.steps))
    res = dict(gpu=gpu_info(), rounds=a.rounds, decode_steps=a.steps, hbm_peak_bytes_per_s=HBM_PEAK)
    for name, rs in rounds.items():
        res[name] = {k: float(np.median([r[k] for r in rs])) for k in rs[0]}
        res[name + "_spread"] = {k: [float(min(r[k] for r in rs)), float(max(r[k] for r in rs))] for k in rs[0]}
    res["fp16_over_bf16"] = {k: res["fp16"][k] / res["bf16"][k] for k in res["bf16"] if k.endswith("_ms") or "per_" in k}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
