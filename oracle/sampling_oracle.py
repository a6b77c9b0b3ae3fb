"""CPU restatement of the sampled decoding of the SEAL VQA LLM (vstar_b200/csrc/sampling.cu, vsb_sample_rows_f32).

The reference samples with transformers' `sample()` (transformers 4.31, `generate(do_sample=True)` from
`vstar_bench_eval.py:97`): TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper -> multinomial(softmax).  The chain
here, step by step:

  1. v = dtype(float(dtype(x)) / float32(T)): the logits are the lm_head output in the model dtype (not upcast), divided as
     torch divides a half / bfloat16 tensor by a Python scalar.
  2. top-k (k > 0): keep v >= the k-th largest v, so every token tied with the k-th value survives.
  3. probabilities e = exp(v - max) in float64 (exactly 1 for the max); top-p (top_p < 1): in descending order (ties by
     ascending id) position j is kept while the mass at and after it, over the total, exceeds 1 - top_p (HF's ascending
     cumsum with `cumsum <= 1 - top_p` removed); position 0 is always kept.
  4. inverse CDF over the kept tokens in that order at u = 53-bit uniform from Philox4x32-10(key = seed, ctr = (step,0,0,0)).

Every decision comes with its margin: the distance of each top-p mass from 1 - top_p, and of u from the nearest CDF edge.
A summation order other than this one can only flip a decision whose margin is at the level of its rounding.
"""
from __future__ import annotations

import numpy as np
import torch

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF


def philox4x32_10(ctr, key):
    """Random123's philox4x32 with 10 rounds: ctr 4 x uint32, key 2 x uint32 -> 4 x uint32 (Python ints)"""
    c0, c1, c2, c3 = (int(x) & MASK for x in ctr)
    k0, k1 = (int(x) & MASK for x in key)
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
        p0, p1 = M0 * c0, M1 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & MASK, p1 & MASK, ((p0 >> 32) ^ c3 ^ k1) & MASK, p0 & MASK
    return c0, c1, c2, c3


def uniform(seed, step):
    """u in [0, 1) with 53 random bits: key = the 64-bit seed (low word first), counter = (step, 0, 0, 0)"""
    s = int(seed) & 0xFFFFFFFFFFFFFFFF
    x = philox4x32_10((int(step), 0, 0, 0), (s & MASK, s >> 32))
    return ((x[0] >> 5) * 67108864.0 + (x[1] >> 6)) / 9007199254740992.0


def scale(logits, temperature, dtype):
    """step 1: fp32 logits [.., n] -> dtype(float(dtype(x)) / T) as float32"""
    x = torch.as_tensor(logits, dtype=torch.float32).to(dtype).float()
    return (x / torch.tensor(float(temperature), dtype=torch.float32)).to(dtype).float()


def _order(v):
    """indices in descending v, ties by ascending id (-0 == +0)"""
    v = np.asarray(v, dtype=np.float64) + 0.0
    return np.lexsort((np.arange(v.size), -v))


def sample_row(logits, temperature, top_k, top_p, dtype, seed, step):
    """one row -> dict(token, margin, p_margin, u_margin, kept (ids in sampling order), probs (their renormalised
    probabilities), u)"""
    v = scale(logits, temperature, dtype).numpy().astype(np.float64)
    n = v.size
    order = _order(v)
    if top_k and top_k < n:
        tau = v[order[max(int(top_k), 1) - 1]]
        order = order[v[order] >= tau]
    vs = v[order]
    m = vs[0]
    with np.errstate(invalid="ignore"):
        e = np.where(vs == m, 1.0, np.exp(vs - m))
    p_margin = np.inf
    J = e.size
    if top_p is not None and float(np.float32(top_p)) < 1.0:
        thr = 1.0 - float(np.float32(top_p))
        E = e.sum()
        after = np.cumsum(e[::-1])[::-1] / E               # mass at and after each position
        keep = after > thr
        keep[0] = True
        J = int(keep.sum())
        assert keep[:J].all(), "top-p keeps a prefix of the descending order"
        if e.size > 1:
            p_margin = float(np.abs(after[1:] - thr).min())
    cdf = np.cumsum(e[:J])
    cdf = cdf / cdf[-1]
    u = uniform(seed, step)
    j = min(int(np.searchsorted(cdf, u, side="right")), J - 1)
    lo = cdf[j - 1] if j else 0.0
    u_margin = float(min(u - lo, cdf[j] - u))
    return dict(token=int(order[j]), margin=min(p_margin, u_margin), p_margin=p_margin, u_margin=u_margin, kept=order[:J],
                probs=np.diff(np.concatenate([[0.0], cdf])), u=u)


def sample_rows(logits, temperature, top_k, top_p, dtype, seeds, step):
    """rows [B, n] -> (tokens int64 [B], margins float64 [B])"""
    rows = [sample_row(logits[b], temperature, top_k, top_p, dtype, seeds[b], step) for b in range(len(seeds))]
    return np.array([r["token"] for r in rows], dtype=np.int64), np.array([r["margin"] for r in rows])


def warp_mask(logits, temperature, top_k, top_p, dtype):
    """bool [n]: the tokens left with a finite score after the three warpers (what `sample()` can draw from, -inf logits
    aside), with the top-p margin -> (mask, p_margin)"""
    r = sample_row(logits, temperature, top_k, top_p, dtype, 0, 0)
    mask = np.zeros(torch.as_tensor(logits).numel(), dtype=bool)
    mask[r["kept"]] = True
    return mask, r["p_margin"]
