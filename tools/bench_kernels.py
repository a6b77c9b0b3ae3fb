"""Micro-benchmarks of the hot kernels (CUDA events, L2 flushed between iterations)."""
import json
import sys
import os
import math

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from vstar_b200 import ops, _lib

BF = torch.bfloat16
flush = torch.empty(256 * 1024 * 1024, dtype=torch.int8, device="cuda") if torch.cuda.is_available() else None


def timeit(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    res = []
    shapes = [(2560, 12288, 4096, "qkv B=8"), (2560, 4096, 4096, "o_proj B=8"), (2560, 22016, 4096, "gate_up B=8"),
              (2560, 4096, 11008, "down B=8"), (20480, 4096, 4096, "o_proj B=64"), (20480, 22016, 4096, "gate_up B=64"),
              (320, 4096, 4096, "o_proj B=1"), (8, 4096, 4096, "decode B=8"), (8, 22016, 4096, "decode gate_up B=8"),
              (18440, 2304, 768, "owl qkv B=8"), (18440, 3072, 768, "owl fc1 B=8"), (2056, 4096, 1024, "clip fc1 B=8"),
              (8192, 8192, 8192, "square 8k")]
    for M, N, K, name in shapes:
        a = torch.randn(M, K, device="cuda").to(BF)
        w = (torch.randn(N, K, device="cuda") / math.sqrt(K)).to(BF)
        out = torch.empty(M, N, dtype=BF, device="cuda")
        ms = timeit(lambda: ops.gemm(a, w, out=out))
        ms_t = timeit(lambda: torch.matmul(a, w.t(), out=out))
        tf = 2 * M * N * K / ms / 1e9
        var = {}
        for tag, bn in (("tile_256", 256), ("tile_128", 128)):
            _lib.call("vsb_gemm_set_tuning", bn, 0)
            var[tag] = round(2 * M * N * K / timeit(lambda: ops.gemm(a, w, out=out)) / 1e9, 1)
        _lib.call("vsb_gemm_set_tuning", 0, 0)
        res.append(dict(kernel="gemm", name=name, M=M, N=N, K=K, ms=ms, tflops=tf, torch_ms=ms_t, torch_tflops=2 * M * N * K / ms_t / 1e9, variants=var))
        print(res[-1], flush=True)
    for B, H, S, D, causal, name in [(8, 32, 320, 128, True, "llama prefill B=8"), (8, 12, 2305, 64, False, "owl B=8"),
                                     (8, 16, 257, 64, False, "clip B=8"), (64, 32, 320, 128, True, "llama prefill B=64"),
                                     (32, 12, 2305, 64, False, "owl B=32")]:
        qkv = torch.randn(B * S, 3 * H * D, device="cuda").to(BF)
        out = torch.empty(B * S, H * D, dtype=BF, device="cuda")
        fl = 4 * B * H * S * S * D * (0.5 if causal else 1.0)
        var = {}
        for tag, impl in (("mma_sync", 1), ("wgmma", 2), ("wgmma_1wg", 3)):
            _lib.call("vsb_attn_set_impl", impl)
            var[tag] = round(fl / timeit(lambda: ops.attn_fused_qkv(qkv, B, S, H, D, causal, D ** -0.5, out=out)) / 1e9, 1)
        _lib.call("vsb_attn_set_impl", 0)
        ms = timeit(lambda: ops.attn_fused_qkv(qkv, B, S, H, D, causal, D ** -0.5, out=out))
        res.append(dict(kernel="flash_attn", name=name, ms=ms, tflops=fl / ms / 1e9, variants=var))
        print(res[-1], flush=True)
    for rows, cols in [(2560, 4096), (18440, 768)]:
        x = torch.randn(rows, cols, device="cuda").to(BF)
        w = torch.ones(cols, device="cuda").to(BF)
        y = torch.empty_like(x)
        ms = timeit(lambda: ops.rmsnorm(x, w, 1e-6, out=y))
        res.append(dict(kernel="rmsnorm", rows=rows, cols=cols, ms=ms, gbs=rows * cols * 4 / ms / 1e6))
        print(res[-1], flush=True)
    os.makedirs("bench_out", exist_ok=True)
    json.dump(res, open("bench_out/bench_kernels.json", "w"), indent=1)


if __name__ == "__main__":
    main()
