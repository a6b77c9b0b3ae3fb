"""Beam search of the SEAL VQA LLM's reference `generate(num_beams=k, do_sample=False)` restated on a per-step logits callback,
in plain Python and torch (fp32 / fp64), with the margin of every decision.

The reference pins transformers 4.31.0 (requirements.txt); the rules below are restated from 4.31's `beam_search`,
`BeamSearchScorer` and `BeamHypotheses` with length_penalty, early_stopping, one returned sequence and no logits processors.
That source is not part of this repository and the installed transformers (5.x) differs in one rule: it leaves the prompt out
of a hypothesis' length.  These rules follow 4.31, not the installed version:
  - step scores: logp = dtype(log_softmax(dtype(logits))) (the reference's fp16 logits; bf16 for a bf16 engine), here computed
    in fp64 and rounded once to dtype (torch computes x - max - log sum exp(x - max) in fp32: the two agree except where the
    unrounded value lies within about one fp32 ulp of a dtype rounding midpoint, reported as `round` margins);
    candidate score = fp32(logp) + beam score in fp32;
  - the first step takes its candidates from the one prompt row (4.31 starts the beam scores at [0, -1e9, ...] over k copies);
  - candidates: the 2k largest over k * V, descending, ties by ascending beam * V + token (torch.topk leaves the order of
    equal values unspecified; this tie rule is the engine's);
  - process(): an eos candidate of rank >= k is skipped, one of rank < k is offered as a hypothesis (the beam's ids without the
    eos, its score with the eos log-prob); any other candidate becomes a running beam until k exist, in rank order;
  - hypothesis score = sum_logprobs / len(hyp) ** length_penalty, len = prompt ids (one id per <image> / <object>) + generated;
  - BeamHypotheses.add: worst starts at 1e9; insert when fewer than k are kept or score > worst; at k + 1 delete the lowest;
  - is_done(best, cur_len): best = max of the step's 2k scores, cur_len = input_ids length before the new token; False while
    fewer than k are kept; early_stopping True: done; False: worst >= best / cur_len ** lp; "never": the same with max_length
    in place of cur_len when lp > 0;
  - the loop ends when the request is done, at prompt_len + max_new_tokens, or when `stop` fires on the running beams;
  - finalize: the open beams of a request that is not done are added with their running scores; the pick is
    sorted(beams, key=score).pop() (on a tie the later entry wins); the output is that hypothesis plus one eos when it is
    shorter than max_length.
"""
from __future__ import annotations

import numpy as np
import torch

PROBES = (1e-4, 1e-5, 1e-6, 1e-7, 1e-8, 1e-9)


def log_probs(logits, dtype):
    """fp32 logits [n, V] -> (logp fp32 [n, V] rounded to dtype, the unrounded fp64 values)"""
    x = torch.as_tensor(logits).float().to(dtype).double()
    m = x.max(-1, keepdim=True).values
    y = x - m - torch.log(torch.exp(x - m).sum(-1, keepdim=True))
    return y.to(dtype).float(), y


def round_margin(y, dtype):
    """the largest probe d of PROBES with dtype(y - d) == dtype(y + d) for every entry of y (fp64), 0 when none holds"""
    for d in PROBES:
        if torch.equal((y - d).to(dtype), (y + d).to(dtype)):
            return d
    return 0.0


def candidates(logits, beam_scores, k, dtype):
    """one step: fp32 logits [k_in, V] of the running beams, their scores (floats) -> dict(
       cand = the 2k (score, token, beam) in rank order, scores as Python floats of the fp32 sums,
       select = score gap between the 2k-th and the (2k+1)-th candidate (inf when there is none),
       round = round_margin over every candidate that could reach the 2k-th score)"""
    logp, y = log_probs(logits, dtype)
    sc = torch.tensor(beam_scores, dtype=torch.float32)
    s = (logp + sc[:, None]).reshape(-1)                           # fp32 sums
    V = logp.shape[1]
    sd = s.double().numpy()
    order = np.lexsort((np.arange(sd.size), -sd))                  # score desc, flat index asc
    n = 2 * k
    top = order[:n]
    cand = [(float(sd[f]), int(f % V), int(f // V)) for f in top]
    with np.errstate(invalid="ignore"):                            # -inf - -inf: no gap to report
        select = float(sd[top[-1]] - sd[order[n]]) if sd.size > n else float("inf")
    select = float("inf") if np.isnan(select) else select
    # entries whose score could reach the 2k-th under a perturbation of the unrounded log-prob
    up = ((y + PROBES[0]).to(dtype).float() + sc[:, None]).reshape(-1)
    near = up >= s[top[-1]]
    rm = round_margin(y.reshape(-1)[near], dtype) if bool(near.any()) else PROBES[0]
    return dict(cand=cand, select=select, round=rm)


class Hypotheses:
    def __init__(self, k, lp, early_stopping, max_length):
        self.k, self.lp, self.es, self.max_length = k, lp, early_stopping, max_length
        self.beams = []
        self.worst = 1e9

    def add(self, ids, sum_logprobs, length):
        """-> margin of the decision: |score - worst| when the list is full, else inf"""
        score = sum_logprobs / (length ** self.lp)
        margin = abs(score - self.worst) if len(self.beams) >= self.k else float("inf")
        if len(self.beams) < self.k or score > self.worst:
            self.beams.append((score, list(ids)))
            if len(self.beams) > self.k:
                ranked = sorted((s, i) for i, (s, _) in enumerate(self.beams))
                del self.beams[ranked[0][1]]
                self.worst = ranked[1][0]
            else:
                self.worst = min(score, self.worst)
        return margin

    def is_done(self, best, cur_len):
        """-> (done, margin)"""
        if len(self.beams) < self.k:
            return False, float("inf")
        if self.es is True:
            return True, float("inf")
        denom = self.max_length if (self.es == "never" and self.lp > 0) else cur_len
        bound = best / denom ** self.lp
        return self.worst >= bound, abs(self.worst - bound)


def beam_search(step_logits, prompt_len, k, max_new_tokens, eos, dtype, length_penalty=1.0, early_stopping=False, stop=None):
    """step_logits(step, beams) -> fp32 logits [len(beams), V] of the token after each running beam (beams: lists of generated
    ids, in beam order; one beam at step 0).  stop(beams) -> bool: a stopping criterion checked after every step.
    -> dict(ids = the new ids the reference's generate returns after the prompt, score, hyp = the chosen hypothesis' ids,
            history = the running beams before every step, margins = dict(select, round, insert, done: lists; pick))"""
    max_length = prompt_len + max_new_tokens
    hyps = Hypotheses(k, length_penalty, early_stopping, max_length)
    beams, scores = [[]], [0.0]
    done = False
    history = []
    mg = dict(select=[], round=[], insert=[], done=[], pick=float("inf"))
    for step in range(max_new_tokens):
        history.append([list(b) for b in beams])
        c = candidates(step_logits(step, beams), scores, k, dtype)
        mg["select"].append(c["select"])
        mg["round"].append(c["round"])
        cur_len = prompt_len + step
        nb, ns = [], []
        for rank, (s, t, b) in enumerate(c["cand"]):
            if t == eos:
                if rank >= k:
                    continue
                mg["insert"].append(hyps.add(beams[b], s, cur_len))
            else:
                nb.append(beams[b] + [t])
                ns.append(s)
            if len(nb) == k:
                break
        beams, scores = nb, ns
        d, m = hyps.is_done(max(x[0] for x in c["cand"]), cur_len)
        mg["done"].append(m)
        done = done or d
        if done or step == max_new_tokens - 1 or (stop is not None and stop(beams)):
            break
    if not done:
        for b, s in zip(beams, scores):
            mg["insert"].append(hyps.add(b, s, prompt_len + len(b)))
    ranked = sorted(hyps.beams, key=lambda x: x[0])
    if len(ranked) > 1:
        mg["pick"] = ranked[-1][0] - ranked[-2][0]
    score, hyp = ranked.pop()
    ids = hyp + [eos] if prompt_len + len(hyp) < max_length else list(hyp)
    return dict(ids=ids, score=score, hyp=hyp, history=history, margins=mg)


def min_margin(res):
    """the smallest decision margin of a beam_search result (selection gaps, insertions, is_done tests, final pick)"""
    m = res["margins"]
    return min([m["pick"]] + m["select"] + m["insert"] + m["done"])
