"""What chunked prefill (DecodeStream(kv_pages=N, prefill_chunk=C)) does to the paged decode stream, on the SEAL VQA LLM at
Vicuna-7B + CLIP-L shapes with random weights, in bf16 and NF4, on the 64-request workload of tools/bench_vqa_stream.py (300-900
prompt rows, 8-512 answer tokens; random weights never emit eos).  A paged stream of 16 slots in the bytes of 16 contiguous
slots (equal_bytes_pages(16)); arms: unchunked, prefill_chunk 256 and 512, alternated `rounds` times (medians and [min, max]).

Per arm: wall time and tokens/s, ms per step, the gaps between consecutive tokens of running requests (host clock around
step(), which ends in a synchronising device-to-host copy; an unchunked admission's prefill counts into the gap of every
running request), time to first token (from the call's start), and whether the tokens equal the unchunked arm's.  Plus one
kernel line: vsb_attn_chunk_paged over a 601-row prompt in chunks of 256 against one vsb_flash_attn of the whole prompt (CUDA
events, 7B attention shapes).  The GPU name and power limit are read in the same run.

    python tools/bench_vqa_stream_chunked.py [--requests 64] [--rounds 2] [--dtypes bf16,nf4] [--out results.json]
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
from vstar_b200.vqa import VQAEngine, VQAWeights

SLOTS = 16
CHUNKS = (256, 512)


def run(eng, reqs, lens, kv_pages, chunk=None):
    """every request through one paged stream, admitted in order as its slot and pages free -> (tokens, stats)"""
    T = [eng.spliced_length(r[0], 0, r[3]) for r in reqs]
    outs = [None] * len(reqs)
    kw = {} if chunk is None else dict(prefill_chunk=chunk)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    st = eng.decode_stream(SLOTS, max_positions=POSITIONS, eos_token_id=-1, kv_pages=kv_pages, **kw)
    owner, nxt, t_step, gaps, ttft, last = {}, 0, 0.0, [], [None] * len(reqs), {}

    def admit():
        nonlocal nxt
        while nxt < len(reqs) and st.free_slots >= 1 and st.pages.need(T[nxt], lens[nxt]) <= st.pages.free_pages:
            r = st.admit(reqs[nxt], lens[nxt])
            owner[r.id] = nxt
            if r.tokens:                                      # unchunked: the first token comes with the admission
                torch.cuda.synchronize()
                now = time.perf_counter()
                ttft[nxt], last[r.id] = now - t0, now
            nxt += 1
    admit()
    remaining = len(reqs)
    while remaining:
        t1 = time.perf_counter()
        done = st.step()                                      # ends in the device-to-host copy of the step's tokens
        now = time.perf_counter()
        t_step += now - t1
        for r in st.active + [r for r, _ in done]:
            if r.tokens and r.id not in last:                 # chunked: first token in this step
                ttft[owner[r.id]], last[r.id] = now - t0, now
            elif r.id in last and last[r.id] != now:
                gaps.append(now - last[r.id])
                last[r.id] = now
        for r, toks in done:
            outs[owner[r.id]] = list(toks)
            remaining -= 1
        admit()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    res = dict(wall_s=wall, steps=st.steps, step_s=t_step, gaps_ms=1e3 * np.array(gaps), ttft_s=np.array(ttft, dtype=float))
    st.close()
    torch.cuda.empty_cache()
    return outs, res


def summarise(runs, tokens):
    wall = [r["wall_s"] for r in runs]
    step = [1e3 * r["step_s"] / max(1, r["steps"]) for r in runs]
    g = runs[int(np.argsort(wall)[len(wall) // 2])]
    q = lambda a, p: float(np.percentile(a, p))
    return dict(wall_s=float(np.median(wall)), wall_s_spread=[min(wall), max(wall)], tokens_per_s=tokens / float(np.median(wall)),
                tokens_per_s_spread=[tokens / max(wall), tokens / min(wall)], ms_per_step=float(np.median(step)),
                ms_per_step_spread=[min(step), max(step)], steps=runs[0]["steps"],
                token_gap_ms=dict(p50=q(g["gaps_ms"], 50), p99=q(g["gaps_ms"], 99), max=float(g["gaps_ms"].max())),
                ttft_s=dict(p50=q(g["ttft_s"], 50), p99=q(g["ttft_s"], 99), max=float(g["ttft_s"].max())))


def kernel_line(dt, T=601, C=256, H=32, D=128, reps=50):
    """vsb_attn_chunk_paged over the prompt in chunks of C (one launch per chunk, as the stream runs it) against one causal
    vsb_flash_attn of all T rows: device ms per prompt"""
    HD, P = H * D, PAGE_ROWS
    n_pages = -(-T // P)
    seq = (torch.randn(T, 3 * HD, device="cuda") * 0.5).to(dt)
    pool = torch.empty((n_pages, P, 2 * HD), dtype=dt, device="cuda")
    pool.view(-1, 2 * HD)[:T] = seq[:, HD:]
    table = torch.arange(n_pages, dtype=torch.int32, device="cuda").view(1, -1)
    out = torch.empty((T, HD), dtype=dt, device="cuda")
    segs = [(lo, min(C, T - lo)) for lo in range(0, T, C)]
    segt = [torch.tensor([[0], [lo], [n]], dtype=torch.int32, device="cuda") for lo, n in segs]

    def chunked():
        for (lo, n), s in zip(segs, segt):
            ops.attn_chunk_paged(seq[lo:lo + n, :HD], pool, table, out[lo:lo + n], H, D, D ** -0.5, s)

    def flash():
        ops.flash_attn(seq, seq[:, HD:], seq[:, 2 * HD:], out, 1, H, T, T, D, True, D ** -0.5, T * 3 * HD, 3 * HD, T * 3 * HD, 3 * HD,
                       T * 3 * HD, 3 * HD, T * HD, HD)
    res = {}
    for _ in range(2):                                        # alternated; the second pass is kept
        for name, fn in (("flash_attn_ms", flash), ("chunk_paged_ms", chunked)):
            fn()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                fn()
            b.record()
            torch.cuda.synchronize()
            res[name] = a.elapsed_time(b) / reps
    want = torch.empty_like(out)
    flash()
    want.copy_(out)
    chunked()
    torch.cuda.synchronize()
    return dict(prompt_rows=T, chunk=C, heads=H, head_dim=D, launches=len(segs), **res, same_bits=bool(torch.equal(out, want)))


def bench_dtype(make_weights, n, rounds):
    eng = VQAEngine(make_weights(), max_tokens=POSITIONS)
    reqs, lens = workload(n)
    reqs = [(ids, img.to(eng.dtype).cuda(), c, il, ol) for ids, img, c, il, ol in reqs]
    tokens = sum(lens)
    pages = equal_bytes_pages(SLOTS)
    arms = {"unchunked": None, **{f"chunk_{c}": c for c in CHUNKS}}
    for c in arms.values():                                   # warm-up of every shape family of every arm
        run(eng, reqs[:6], [6] * 6, pages, c)
    res, outs = {a: [] for a in arms}, {}
    for _ in range(rounds):
        for a, c in arms.items():
            outs[a], r = run(eng, reqs, lens, pages, c)
            res[a].append(r)
    out = dict(requests=n, generated_tokens=tokens, slots=SLOTS, kv_pages=pages, page_rows=PAGE_ROWS, positions=POSITIONS)
    for a in arms:
        out[a] = dict(summarise(res[a], tokens), same_tokens_as_unchunked=outs[a] == outs["unchunked"])
    out["kernel_601_rows_chunks_256"] = kernel_line(eng.dtype)
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
        raise SystemExit("bench_vqa_stream_chunked needs a CUDA GPU (nothing is measured on the CPU)")
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
