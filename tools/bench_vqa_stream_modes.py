"""Sampled and beam-search answers on the decode stream (DecodeStream.admit(temperature=, num_beams=)) against the static batch of
generate_batch with the same settings, on the SEAL VQA LLM at Vicuna-7B + CLIP-L shapes with random weights, in bf16 and NF4.

Workload: the 64 requests of tools/bench_vqa_stream.py (SEAL-shaped prompts of 300-900 rows, answer lengths log-uniform over
8-512 tokens; random weights never emit eos, so every request runs to its own max_new_tokens).
  * sampled (temperature 0.7, top_k 50, top_p 0.9; request i with seed i) at 8, 16 and 32 slots: static = generate_batch over
    consecutive chunks of `slots` requests, each chunk run to its longest budget and every answer cut to its own; stream = one
    decode stream with `slots` slots;
  * beam search (k = 4) at 16 and 32 slots, i.e. 4 and 8 requests in flight: static = generate_batch(num_beams=4) over chunks of
    slots / 4 requests (each chunk searches to its longest budget); stream = one decode stream, a request admitted when 4
    slots are free;
  * greedy stream at 16 slots with the parent commit's step (ParentGreedyStream, argmax and its copy only) and with today's,
    so a greedy-only stream is shown not to have slowed down.
Reported per (dtype, mode, slots): wall time, generated tokens/s, mean occupied slots (rows) per decode step, ms per decode
step (decode time without the CLIP + prefill work), medians over rounds that alternate static and stream; and how often the
stream's answer equals the static one (sampled: every draw is keyed by (seed, step), so they agree wherever the two decodes'
logits round alike; beam: the static chunk searches to its longest budget, which changes a hypothesis' max_length).
torch.profiler, in a run of its own: the sampler, candidate and row-copy kernels' shares of the GPU time of 32 stream steps.
The GPU name, power limit and clocks are read in the same run.

    python tools/bench_vqa_stream_modes.py [--requests 64] [--rounds 2] [--out results.json]
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
from tools.bench_vqa_stream import Timer, free_engine_cache, summarise, workload
from vstar_b200 import ops, synth
from vstar_b200.config import VSMConfig
from vstar_b200.vqa import DecodeStream, VQAEngine, VQAWeights

SAMPLE = dict(temperature=0.7, top_k=50, top_p=0.9)
SAMPLE_SLOTS = (8, 16, 32)
BEAM_K = 4
BEAM_SLOTS = (16, 32)
GREEDY_SLOTS = 16


class ParentGreedyStream(DecodeStream):
    """the greedy step as the parent commit ran it (every row argmax'd, its tokens read by one copy), for the before/after row"""

    def step(self):
        self._check_open()
        done, self._finished = [(r, r.tokens) for r in self._finished], []
        act = self.active
        if not act:
            return done
        e, c = self.engine, self.engine.cfg
        B = len(act)
        lens = [r.prompt_len + len(r.tokens) - 1 for r in act]
        meta = torch.tensor([[r.slot for r in act], lens, lens], dtype=torch.int32).to(e.dev)
        ids = torch.tensor([r.tokens[-1] for r in act], dtype=torch.int64).to(e.dev)
        x = ops.gather_rows(ids, e.w.embed)
        ops.llama_layers_slots(e._layer_table, len(e.w.layers), x, self._cache, c.rms_eps, e.w.rope_cos, e.w.rope_sin, self._scratch,
                               meta[0], meta[1], meta[2], max(lens), c.n_heads, c.intermediate,
                               norm_folded=getattr(e.w, "fold_norms", False), deq_scratch=self._deq)
        hn = ops.rmsnorm(x, e.w.final_norm, c.rms_eps)
        logits = ops.gemm(hn, e.w.lm_head, out_dtype=torch.float32)
        nxt = ops.argmax_rows(logits)[0].tolist()
        self.last_logits = (act, logits)
        self.steps += 1
        self.occupied += B
        for r, t in zip(act, nxt):
            r.tokens.append(int(t))
            if self._ended(r):
                r.done = True
                self._slots[r.slot] = None
                done.append((r, r.tokens))
        return done


def run_static(eng, reqs, lens, slots, mode):
    per = slots // BEAM_K if mode == "beam" else slots
    rows = BEAM_K if mode == "beam" else 1
    outs, steps = [], 0
    tm = Timer(eng, ["build_embeds_batch", "prefill_ragged"])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(0, len(reqs), per):
        chunk, budgets = reqs[i:i + per], lens[i:i + per]
        if mode == "beam":
            o = eng.generate_batch(chunk, max_new_tokens=max(budgets), eos_token_id=-1, num_beams=BEAM_K)
        else:
            o = eng.generate_batch(chunk, max_new_tokens=max(budgets), eos_token_id=-1, seeds=list(range(i, i + len(chunk))), **SAMPLE)
        outs += [x[:n] for x, n in zip(o, budgets)]
        steps += max(budgets) - 1
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    tm.remove()
    free_engine_cache(eng)
    return outs, dict(wall_s=wall, steps=steps, decode_s=wall - tm.t, occupied=rows * (sum(lens) - len(lens)))


def run_stream(eng, reqs, lens, slots, mode, cls=DecodeStream):
    outs = [None] * len(reqs)
    need = BEAM_K if mode == "beam" else 1
    longest = max(eng.spliced_length(r[0], 0, r[3]) + n for r, n in zip(reqs, lens))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    st = cls(eng, slots, longest, -1)
    owner, nxt, t_step = {}, 0, 0.0

    def admit():
        nonlocal nxt
        kw = dict(num_beams=BEAM_K) if mode == "beam" else dict(seed=nxt, **SAMPLE) if mode == "sample" else {}
        owner[st.admit(reqs[nxt], lens[nxt], **kw).id] = nxt
        nxt += 1

    while nxt < len(reqs) and st.free_slots >= need:
        admit()
    remaining = len(reqs)
    while remaining:
        t1 = time.perf_counter()
        done = st.step()                                      # ends in the device-to-host copy of the step's selections
        t_step += time.perf_counter() - t1
        for r, toks in done:
            outs[owner[r.id]] = toks[:lens[owner[r.id]]]
            remaining -= 1
        while nxt < len(reqs) and st.free_slots >= need:
            admit()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    res = dict(wall_s=wall, steps=st.steps, decode_s=t_step, occupied=st.occupied)
    st.close()
    return outs, res


def kernel_shares(eng, reqs, mode, slots=16, steps=32):
    """GPU-time shares of the selection kernels over `steps` stream steps with every slot busy"""
    from torch.profiler import ProfilerActivity, profile
    need = BEAM_K if mode == "beam" else 1
    st = eng.decode_stream(slots, max_positions=1024, eos_token_id=-1)
    for i, r in enumerate(reqs[:slots // need]):
        st.admit(r, steps + 2, **(dict(num_beams=BEAM_K) if mode == "beam" else dict(seed=i, **SAMPLE)))
    st.step()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            st.step()
        torch.cuda.synchronize()
    st.close()
    names = dict(sampler="sample_rows_kernel", candidates="beam_candidates_kernel", row_copy="copy_cache_rows_kernel")
    us = {k: 0.0 for k in names}
    tot = 0.0
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if t <= 0:
            continue
        tot += t
        for k, pat in names.items():
            if pat in e.key:
                us[k] += t
    out = dict(mode=mode, slots=slots, steps=steps, gpu_us_per_step=tot / steps)
    for k in names:
        out[f"{k}_us_per_step"] = us[k] / steps
        out[f"{k}_share"] = us[k] / tot
    return out


def bench_dtype(make_weights, n, rounds):
    eng = VQAEngine(make_weights(), max_tokens=1024)
    reqs, lens = workload(n)
    reqs = [(ids, img.to(eng.dtype).cuda(), c, il, ol) for ids, img, c, il, ol in reqs]
    total = sum(lens)
    out = dict(requests=n, generated_tokens=total)
    for mode in ("sample", "beam"):                          # warm-up: every kernel family of both modes
        run_static(eng, reqs[:4], [4] * 4, 4 if mode == "sample" else 8, mode)
        run_stream(eng, reqs[:4], [4] * 4, 8, mode)
    cases = [("sample", s) for s in SAMPLE_SLOTS] + [("beam", s) for s in BEAM_SLOTS]
    for mode, slots in cases:
        st_runs, sm_runs = [], []
        for _ in range(rounds):
            o_static, r = run_static(eng, reqs, lens, slots, mode)
            st_runs.append(r)
            o_stream, r = run_stream(eng, reqs, lens, slots, mode)
            sm_runs.append(r)
        s, m = summarise(st_runs, total, slots, lens), summarise(sm_runs, total, slots, lens)
        out[f"{mode}_slots{slots}"] = dict(static=s, stream=m, stream_speedup_wall=s["wall_s"] / m["wall_s"],
                                           same_answer=sum(a == b for a, b in zip(o_static, o_stream)) / n)
        print(json.dumps({f"{mode}_slots{slots}": out[f"{mode}_slots{slots}"]}), flush=True)
    before, after = [], []
    for _ in range(rounds):
        o_before, r = run_stream(eng, reqs, lens, GREEDY_SLOTS, "greedy", cls=ParentGreedyStream)
        before.append(r)
        o_after, r = run_stream(eng, reqs, lens, GREEDY_SLOTS, "greedy")
        after.append(r)
    b, a = summarise(before, total, GREEDY_SLOTS, lens), summarise(after, total, GREEDY_SLOTS, lens)
    out[f"greedy_slots{GREEDY_SLOTS}"] = dict(parent_step=b, this_step=a, wall_ratio=a["wall_s"] / b["wall_s"],
                                              same_answer=sum(x == y for x, y in zip(o_before, o_after)) / n)
    out["profile"] = [kernel_shares(eng, reqs, "sample"), kernel_shares(eng, reqs, "beam")]
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
        raise SystemExit("bench_vqa_stream_modes needs a CUDA GPU (nothing is measured on the CPU)")
    res = dict(gpu_before=gpu_info(), rounds=a.rounds)
    cfg = VSMConfig()
    shapes = synth.vqa_state_dict_shapes(cfg)
    get = lambda n: synth.synthetic_tensor(n, shapes[n], seed=4321, device="cuda")
    makers = dict(bf16=lambda: VQAWeights(cfg, get, dtype=torch.bfloat16),
                  nf4=lambda: VQAWeights(cfg, get, dtype=torch.float16, quant="nf4"))
    with torch.inference_mode():
        for name in a.dtypes.split(","):
            res[name] = bench_dtype(makers[name], a.requests, a.rounds)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
