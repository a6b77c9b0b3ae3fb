"""The wgmma tile GEMM at the shapes and with the epilogues of the headline step (bench.py configs[2]), timed with CUDA events.

Rows (bf16, random data, one H100 per run):
  * Llama-7B prefill projections with their real epilogues, at B = 8 / 32 / 64 crops of 283 rows and at the tail-only shapes
    (B * 5 rows):
      qkv   folded-RMSNorm input (128 partial sums per row), fused RoPE, rows remapped into a [B, 384, 3d] cache at past = 37
      o     in-place residual (x += a Wo^T), row statistics out
      gu    folded-RMSNorm input, SwiGLU
      down  K = 11008, in-place residual, row statistics out
  * the CLIP-L (M = B*257) and OWL-B (M = B*2305) Linears with bias / QuickGELU / residual;
  * a K sweep (256 ... 4096) at the qkv, o and gu shapes of 64 crops and the CLIP qkv shape (bias) of 64 crops.  Time is linear in K: the slope is the main loop's rate, the
    intercept the cost every tile pays whatever K is (mostly the epilogue), reported per wave of tiles as well.
Every row also times torch.matmul (cuBLAS) on the same M, N, K without an epilogue, as a reference for the card; cuBLAS is not
used by the product.

    python tools/bench_gemm_epilogue.py [--lib path/to/libvstar_b200.so] [--out results.json] [--quick]

--lib loads another build of the library (for example the parent commit's) through the same Python wrappers, so two builds can be
timed on the same card by alternating runs.  The card's name, power limit and max SM clock are read in the same run.
"""
import argparse
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from vstar_b200 import _lib

BF = torch.bfloat16
D, INTER, T_CROP, T_MAX, PAST = 4096, 11008, 283, 384, 37
BM = 128


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().split("\n")[0]
    except (OSError, subprocess.SubprocessError):
        q = ""
    return dict(device=torch.cuda.get_device_name(), nvidia_smi=q, sms=torch.cuda.get_device_properties(0).multi_processor_count)


def tile_bn(M, N, sms, rope=False, swiglu=False):
    """the tile width gemm_dispatch (gemm_tcgen05.cu) picks for an M x N tile-kernel GEMM"""
    if rope:
        return 256
    bn = 64
    if N > 64:
        tm, best = -(-M // BM), None
        for c in (256, 128, 64):
            if c == 256 and not swiglu:
                continue
            if c == 64 and N > 512:
                continue
            cost = -(-(tm * -(-N // c)) // sms) * c
            if best is None or cost < best:
                best, bn = cost, c
    if bn == 64 and -(-M // BM) * -(-N // 64) <= sms // 2 and N >= 64:
        bn = 32
    return bn


def time_ms(fn, target_ms=30.0, windows=5):
    """median over `windows` event-timed windows of the per-call time; each window runs enough calls to last ~target_ms"""
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    reps = max(2, min(2000, int(math.ceil(target_ms / max(a.elapsed_time(b), 1e-3)))))
    out = []
    for _ in range(windows):
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b) / reps)
    return float(np.median(out)), float(min(out)), float(max(out))


def stream():
    return torch.cuda.current_stream().cuda_stream


class Bufs:
    """device buffers sized for the largest shape, shared by every row (random bf16 data, positive row statistics)"""

    def __init__(self, Bmax):
        g = torch.Generator(device="cuda").manual_seed(0)
        rows = Bmax * T_CROP
        self.x = torch.randn(rows, INTER, device="cuda", generator=g).to(BF)        # also the attention output / SwiGLU output
        self.y = torch.randn(rows, INTER, device="cuda", generator=g).to(BF)
        self.cache = torch.zeros(Bmax * T_MAX, 3 * D, dtype=BF, device="cuda")
        self.c = torch.empty(rows * 2 * INTER, dtype=BF, device="cuda")                 # cuBLAS output
        self.w = (torch.randn(2 * INTER, INTER, device="cuda", generator=g) / 64).to(BF)
        self.bias = (torch.randn(2 * INTER, device="cuda", generator=g) / 8).to(BF)
        self.sq_in = (torch.rand(D // 32, rows, device="cuda", generator=g) + 0.5) * (32.0 / 1.0)
        self.sq_out = torch.empty(D // 32, rows, device="cuda")
        pos = torch.arange(2048, device="cuda", dtype=torch.float32)[:, None]
        inv = 1.0 / (10000.0 ** (torch.arange(0, 128, 2, device="cuda", dtype=torch.float32) / 128))
        ang = torch.cat([pos * inv, pos * inv], 1)[:, :64]
        self.cos, self.sin = ang.cos().to(BF).contiguous(), ang.sin().to(BF).contiguous()


def llama_calls(bf, B, rows_per_seq):
    """(name, M, N, K, rope, fn) of the four prefill projections of one layer at B sequences of rows_per_seq rows"""
    M = B * rows_per_seq
    x, y, w, sq_in, sq_out = bf.x, bf.y, bf.w, bf.sq_in, bf.sq_out
    s = stream

    def qkv():
        _lib.call("vsb_gemm_qkv_rope_bf16", x.data_ptr(), D, w.data_ptr(), D, bf.cache.data_ptr(), 3 * D, M, 3 * D, D, rows_per_seq, T_MAX,
                  PAST, sq_in.data_ptr(), D // 32, 1e-6, M, bf.cos.data_ptr(), bf.sin.data_ptr(), None, rows_per_seq, PAST, 128, s())

    def oproj():
        _lib.call("vsb_gemm_rowscale_bf16", y.data_ptr(), D, w.data_ptr(), D, x.data_ptr(), D, M, D, D, None, x.data_ptr(), D, 0, 0, 0, 0,
                  None, 0, 1e-6, sq_out.data_ptr(), M, s())

    def gu():
        _lib.call("vsb_gemm_rowscale_bf16", x.data_ptr(), D, w.data_ptr(), D, y.data_ptr(), INTER, M, 2 * INTER, D, None, None, 0, 4, 0, 0,
                  0, sq_in.data_ptr(), D // 32, 1e-6, None, M, s())

    def down():
        _lib.call("vsb_gemm_rowscale_bf16", y.data_ptr(), INTER, w.data_ptr(), INTER, x.data_ptr(), D, M, D, INTER, None, x.data_ptr(), D,
                  0, 0, 0, 0, None, 0, 1e-6, sq_out.data_ptr(), M, s())

    return [("qkv", M, 3 * D, D, True, qkv), ("o", M, D, D, False, oproj), ("gu", M, 2 * INTER, D, False, gu),
            ("down", M, D, INTER, False, down)]


def vit_calls(bf, name, M, d, inter):
    """(name, M, N, K, rope, fn) of the Linears of one pre-LN ViT block: qkv (bias), o (bias + residual), fc1 (bias + QuickGELU),
    fc2 (bias + residual)"""
    x, y, w, bias = bf.x, bf.y, bf.w, bf.bias

    def lin(a, lda, N, K, out, ldo, epi, res):
        def f():
            _lib.call("vsb_gemm_bf16", a.data_ptr(), lda, w.data_ptr(), K, out.data_ptr(), ldo, M, N, K, bias.data_ptr(),
                      res.data_ptr() if res is not None else None, ldo if res is not None else 0, epi, 0, 0, 0, 0, stream())
        return f

    return [(f"{name}.qkv", M, 3 * d, d, False, lin(x, d, 3 * d, d, y, 3 * d, 0, None)),
            (f"{name}.o", M, d, d, False, lin(y, d, d, d, x, d, 0, x)),
            (f"{name}.fc1", M, inter, d, False, lin(x, d, inter, d, y, inter, 1, None)),
            (f"{name}.fc2", M, d, inter, False, lin(y, inter, d, inter, x, d, 0, x))]


def cublas_fn(bf, M, N, K):
    a, w = bf.x.view(-1)[:M * K].view(M, K), bf.w.view(-1)[:N * K].view(N, K)
    out = bf.c[:M * N].view(M, N)
    return lambda: torch.matmul(a, w.t(), out=out)


def row(bf, sms, name, M, N, K, rope, fn, cublas=True):
    ms, lo, hi = time_ms(fn)
    flops = 2.0 * M * N * K
    bn = tile_bn(M, N, sms, rope, swiglu=name.split(".")[0].split("@")[0] == "gu")
    tiles = -(-M // BM) * -(-N // bn)
    r = dict(name=name, M=M, N=N, K=K, bn=bn, tiles=tiles, waves=-(-tiles // sms), ms=ms, ms_spread=[lo, hi], tflops=flops / ms / 1e9)
    if cublas:
        cms = time_ms(cublas_fn(bf, M, N, K))[0]
        r.update(cublas_ms=cms, cublas_tflops=flops / cms / 1e9)
    print(f"{name:>14s} M={M:6d} N={N:6d} K={K:6d} bn={bn:3d} waves={r['waves']:3d}  {ms:8.3f} ms  {r['tflops']:6.1f} TFLOP/s"
          + (f"   cuBLAS {r['cublas_ms']:8.3f} ms {r['cublas_tflops']:6.1f}" if cublas else ""), file=sys.stderr)
    return r


def k_sweep(bf, sms, which, B, ks):
    pts = []
    for K in ks:
        _, M, N, _, rope, fn = _sweep_call(bf, which, B, K)
        pts.append(row(bf, sms, f"{which}@K={K}", M, N, K, rope, fn, cublas=False))
    K = np.array([p["K"] for p in pts], dtype=np.float64)
    t = np.array([p["ms"] for p in pts])
    slope, icpt = np.polyfit(K, t, 1)
    M, N, waves = pts[0]["M"], pts[0]["N"], pts[0]["waves"]
    return dict(shape=which, M=M, N=N, bn=pts[0]["bn"], waves=waves, points=[(p["K"], p["ms"]) for p in pts], intercept_ms=float(icpt),
                intercept_us_per_wave=float(icpt) * 1e3 / waves, slope_ms_per_k=float(slope),
                main_loop_tflops=2.0 * M * N / (slope * 1e-3) / 1e12)


def _sweep_call(bf, which, B, K):
    """the qkv (folded norm + RoPE + cache remap), o (in-place residual + row statistics), gu (folded norm + SwiGLU) or CLIP
    qkv (bias) GEMM of B crops with its K changed"""
    M = B * T_CROP
    x, y, w = bf.x, bf.y, bf.w
    if which == "qkv":
        def f():
            _lib.call("vsb_gemm_qkv_rope_bf16", x.data_ptr(), K, w.data_ptr(), K, bf.cache.data_ptr(), 3 * D, M, 3 * D, K, T_CROP, T_MAX,
                      PAST, bf.sq_in.data_ptr(), D // 32, 1e-6, M, bf.cos.data_ptr(), bf.sin.data_ptr(), None, T_CROP, PAST, 128,
                      stream())
        return "qkv", M, 3 * D, K, True, f
    if which == "clip.qkv":
        M, N = B * 257, 3 * 1024
        def f():
            _lib.call("vsb_gemm_bf16", x.data_ptr(), K, w.data_ptr(), K, y.data_ptr(), N, M, N, K, bf.bias.data_ptr(), None, 0, 0, 0, 0, 0,
                      0, stream())
        return "clip.qkv", M, N, K, False, f
    if which == "o":
        def f():
            _lib.call("vsb_gemm_rowscale_bf16", y.data_ptr(), K, w.data_ptr(), K, x.data_ptr(), D, M, D, K, None, x.data_ptr(), D, 0, 0, 0,
                      0, None, 0, 1e-6, bf.sq_out.data_ptr(), M, stream())
        return "o", M, D, K, False, f

    def f():
        _lib.call("vsb_gemm_rowscale_bf16", x.data_ptr(), K, w.data_ptr(), K, y.data_ptr(), INTER, M, 2 * INTER, K, None, None, 0, 4, 0, 0, 0,
                  bf.sq_in.data_ptr(), D // 32, 1e-6, None, M, stream())
    return "gu", M, 2 * INTER, K, False, f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="libvstar_b200.so to load instead of the in-tree build")
    ap.add_argument("--out", default=None, help="also write the result JSON here")
    ap.add_argument("--quick", action="store_true", help="B = 8 only and a 3-point K sweep")
    a = ap.parse_args()
    if a.lib:
        _lib.LIB_PATH = os.path.abspath(a.lib)
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm_epilogue needs a CUDA GPU (nothing is measured on the CPU)")
    _lib.load()
    info = gpu_info()
    sms = info["sms"]
    batches = (8,) if a.quick else (8, 32, 64)
    ks = (256, 1024, 4096) if a.quick else (256, 512, 1024, 2048, 4096)
    bf = Bufs(max(batches))
    rows = []
    with torch.inference_mode():
        for B in batches:
            for rps in (T_CROP, 5):
                for name, M, N, K, rope, fn in llama_calls(bf, B, rps):
                    rows.append(row(bf, sms, f"{name}.B{B}" + ("" if rps == T_CROP else ".tail"), M, N, K, rope, fn))
        # ViT row counts within the buffers: CLIP-L at the smallest and largest B, OWL-B (2305 rows per crop) at B = 8
        vit = [c for B in sorted({batches[0], batches[-1]}) for c in vit_calls(bf, f"clip.B{B}", B * 257, 1024, 4096)]
        for name, M, N, K, rope, fn in vit + vit_calls(bf, "owl.B8", 8 * 2305, 768, 3072):
            rows.append(row(bf, sms, name, M, N, K, rope, fn))
        sweeps = [k_sweep(bf, sms, w, max(batches), ks) for w in ("qkv", "o", "gu", "clip.qkv")]
    res = dict(gpu=info, lib=_lib.LIB_PATH, rows=rows, k_sweep=sweeps)
    for s in sweeps:
        print(f"K sweep {s['shape']}: intercept {s['intercept_ms']:.3f} ms ({s['intercept_us_per_wave']:.2f} us per wave of "
              f"{s['waves']}), main loop {s['main_loop_tflops']:.0f} TFLOP/s", file=sys.stderr)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
