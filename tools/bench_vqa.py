"""Latency probes for the two launch-/HBM-bound corners of the path (run on the GPU):
  * SEAL VQA LLM at full size (Vicuna-7B shapes, random init): prefill, greedy decode ms/token, option scoring
    (vstar_bench_eval.py:78-165) and the M=1 decode GEMMs against the HBM roofline (weights are read once per token);
  * one single-crop VSM round (the root round of every search): wall clock vs GPU time vs launches.
Writes bench_out/bench_vqa.json."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from vstar_b200 import _lib, ops, synth
from vstar_b200.config import VSMConfig

BF = torch.bfloat16
res = {}


def ev_time(fn, iters=5, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    gpu, wall = [], []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        wall.append((time.perf_counter() - t0) * 1e3)
        gpu.append(a.elapsed_time(b))
    return float(np.median(gpu)), float(np.median(wall))


def main():
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    cfg = VSMConfig()
    peak = 6569.0
    p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
    if which in ("all", "gemv"):
        out = []
        for name, N, K in [("qkv", 3 * 4096, 4096), ("o", 4096, 4096), ("gate_up", 22016, 4096), ("down", 4096, 11008), ("lm_head", 32004, 4096)]:
            # 4 weight copies (> L2 together) used round-robin inside ONE CUDA graph of 24 launches: no host launch gaps, no L2 reuse
            ws = [(torch.randn(N, K, device="cuda") / 64).to(BF) for _ in range(4)]
            for M in (1, 2, 4, 8, 16):
                a = torch.randn(M, K, device="cuda").to(BF)
                y = torch.empty(M, N, dtype=BF, device="cuda")
                ops.gemm(a, ws[0], out=y)
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    for i in range(24):
                        ops.gemm(a, ws[i % 4], out=y)
                t, _ = ev_time(g.replay, iters=10, warmup=3)
                t /= 24
                out.append(dict(name=name, M=M, N=N, K=K, us=t * 1e3, gbs=N * K * 2 / t / 1e6, frac_hbm=N * K * 2 / t / 1e6 / peak))
                print(out[-1], flush=True)
            del ws
        res["decode_gemms"] = out
    if which in ("all", "vqa"):
        from vstar_b200.vqa import VQAEngine, VQAWeights
        shapes = synth.vqa_state_dict_shapes(cfg)
        w = VQAWeights(cfg, lambda n: synth.synthetic_tensor(n, shapes[n], seed=4321, device="cuda"))
        eng = VQAEngine(w, max_tokens=1536)
        gen = torch.Generator().manual_seed(0)
        image = torch.randn(1, 3, 224, 224, generator=gen).to(BF).cuda()
        crops = torch.randn(2, 3, 224, 224, generator=gen).to(BF).cuda()
        rng = np.random.default_rng(0)
        q = [1] + rng.integers(1000, 30000, 40).tolist() + [-200] + rng.integers(1000, 30000, 30).tolist() + [-300] + \
            rng.integers(1000, 30000, 8).tolist() + [-300] + rng.integers(1000, 30000, 20).tolist()
        il, ol = [False], [True, True]                      # image short (32 rows), 2 objects long (256 rows each)
        x = eng.build_embeds(q, image, crops, il, ol)
        T = x.shape[0]
        g, wl = ev_time(lambda: eng.prefill_embeds(eng.build_embeds(q, image, crops, il, ol)))
        res["vqa_prefill"] = dict(T=T, gpu_ms=g, wall_ms=wl)
        print(res["vqa_prefill"], flush=True)
        n_new = 64
        l0 = _lib.launches
        g, wl = ev_time(lambda: eng.generate(q, image, crops, il, ol, max_new_tokens=n_new, eos_token_id=-1), iters=3, warmup=1)
        launches = (_lib.launches - l0) // 4
        res["vqa_generate"] = dict(T=T, new_tokens=n_new, gpu_ms=g, wall_ms=wl, ms_per_token=(wl - res["vqa_prefill"]["wall_ms"]) / n_new,
                                   launches=launches, hbm_floor_ms_per_token=13.5e9 / (peak * 1e9) * 1e3)
        print(res["vqa_generate"], flush=True)
        opts = [rng.integers(1000, 30000, 6).tolist() for _ in range(4)]
        g, wl = ev_time(lambda: eng.option_losses(q, opts, image, crops, il, ol), iters=3, warmup=1)
        res["vqa_options"] = dict(T=T, options=4, gpu_ms=g, wall_ms=wl)
        print(res["vqa_options"], flush=True)
        for nb in (4, 8, 16):
            reqs = []
            for i in range(nb):
                qi = [1] + rng.integers(1000, 30000, 30 + 3 * i).tolist() + [-200] + rng.integers(1000, 30000, 20 + 5 * i).tolist()
                reqs.append((qi, image, None, [True], None))
            g, wl = ev_time(lambda: eng.generate_batch(reqs, max_new_tokens=n_new, eos_token_id=-1), iters=2, warmup=1)
            g1, wl1 = ev_time(lambda: eng.prefill_ragged([eng.build_embeds(*r) for r in reqs]), iters=2, warmup=1)
            res[f"vqa_generate_batch{nb}"] = dict(B=nb, new_tokens=n_new, wall_ms=wl, prefill_wall_ms=wl1, ms_per_step=(wl - wl1) / n_new,
                                                  tokens_per_s=nb * n_new / ((wl - wl1) / 1e3))
            print(res[f"vqa_generate_batch{nb}"], flush=True)
        del eng, w
        torch.cuda.empty_cache()
    if which in ("all", "round"):
        from vstar_b200.engine import VSMEngine, VSMWeights
        from vstar_b200.vsm import VSM
        from PIL import Image
        shp = synth.state_dict_shapes(cfg)
        weights = VSMWeights(cfg, lambda n: synth.synthetic_tensor(n, shp[n], seed=1234, device="cuda"))
        engine = VSMEngine(weights, max_tokens=384)
        prompt, ans = synth.synthetic_prompt(cfg, n_text=60, seed=0, im_start_index=37)

        class BenchVSM(VSM):
            def _ids(self, question):
                return prompt[0].tolist()

        vsm = BenchVSM(engine=engine, forced_answer_ids=ans.tolist(), frontier_batch=64)
        img = Image.fromarray(np.random.default_rng(0).integers(0, 256, (1024, 1024, 3), dtype=np.uint8), "RGB")
        for nb in (1, 4, 16):
            regions = [(img, (0, 0, 1024, 1024))] * nb
            l0 = _lib.launches
            g, wl = ev_time(lambda: vsm.detect_regions(regions, ["Please locate the mug in this image."] * nb), iters=5, warmup=2)
            res[f"vsm_round_B{nb}"] = dict(gpu_ms=g, wall_ms=wl, launches=(_lib.launches - l0) // 7)
            print(nb, res[f"vsm_round_B{nb}"], flush=True)
    os.makedirs("bench_out", exist_ok=True)
    json.dump(res, open("bench_out/bench_vqa.json", "w"), indent=1)


if __name__ == "__main__":
    main()
