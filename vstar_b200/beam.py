"""Host side of beam search for the SEAL VQA LLM: transformers 4.31's `BeamHypotheses` / `BeamSearchScorer` (length_penalty,
early_stopping, one returned sequence), applied to the candidates vsb_beam_candidates_f32 selects on the device.

Lengths are those of the reference's `input_ids`: the prompt ids (one id per <image> / <object> placeholder) plus the generated
ids, not the spliced embedding rows.  oracle/beam_oracle.py restates the same rules independently for the tests.
"""
from __future__ import annotations

DEFAULT_LENGTH_PENALTY = 1.0       # transformers 4.31 GenerationConfig defaults
DEFAULT_EARLY_STOPPING = False


def check_beams(num_beams, early_stopping):
    if isinstance(num_beams, bool) or not isinstance(num_beams, int) or not 1 <= num_beams <= 16:
        raise ValueError(f"num_beams must be an integer in [1, 16], got {num_beams!r}")
    if early_stopping not in (True, False, "never"):
        raise ValueError(f"early_stopping must be True, False or 'never', got {early_stopping!r}")


class BeamHypotheses:
    """the finished hypotheses of one request (BeamHypotheses of transformers 4.31, list semantics kept)"""

    def __init__(self, num_beams, length_penalty, early_stopping, max_length):
        self.k, self.lp, self.early_stopping, self.max_length = num_beams, length_penalty, early_stopping, max_length
        self.beams = []                                  # [(score, generated ids)] in insertion order
        self.worst_score = 1e9

    def add(self, ids, sum_logprobs, length):
        """length: the hypothesis' input_ids length (prompt ids + generated ids)"""
        score = sum_logprobs / (length ** self.lp)
        if len(self.beams) < self.k or score > self.worst_score:
            self.beams.append((score, list(ids)))
            if len(self.beams) > self.k:
                ranked = sorted((s, i) for i, (s, _) in enumerate(self.beams))
                del self.beams[ranked[0][1]]
                self.worst_score = ranked[1][0]
            else:
                self.worst_score = min(score, self.worst_score)

    def is_done(self, best_sum_logprobs, cur_len):
        if len(self.beams) < self.k:
            return False
        if self.early_stopping is True:
            return True
        if self.early_stopping is False or self.lp <= 0:
            return self.worst_score >= best_sum_logprobs / cur_len ** self.lp
        return self.worst_score >= best_sum_logprobs / self.max_length ** self.lp      # "never", lp > 0


class BeamRequest:
    """running beams and finished hypotheses of one request"""

    def __init__(self, num_beams, prompt_len, max_new_tokens, eos_token_id, length_penalty, early_stopping):
        self.k, self.prompt_len, self.eos = num_beams, prompt_len, eos_token_id
        self.max_length = prompt_len + max_new_tokens
        self.hyps = BeamHypotheses(num_beams, length_penalty, early_stopping, self.max_length)
        self.beams = [[]]                                # generated ids of the running beams, in beam order
        self.scores = [0.0]
        self.done = False

    def process(self, cand):
        """cand: the step's 2k (score, token, beam) in rank order (BeamSearchScorer.process) -> the k new beams as
        (score, token, parent beam) in rank order; finished hypotheses are offered, `done` updated"""
        cur_len = self.prompt_len + len(self.beams[0])
        nxt = []
        for rank, (s, t, b) in enumerate(cand):
            if t == self.eos:
                if rank >= self.k:
                    continue
                self.hyps.add(self.beams[b], s, cur_len)
            else:
                nxt.append((s, t, b))
            if len(nxt) == self.k:
                break
        self.beams = [self.beams[b] + [t] for s, t, b in nxt]
        self.scores = [s for s, t, b in nxt]
        self.done = self.done or self.hyps.is_done(max(c[0] for c in cand), cur_len)
        return nxt

    def finalize(self):
        """-> (new token ids as the reference's generate returns them after the prompt, score of the chosen hypothesis)"""
        if not self.done:
            for ids, s in zip(self.beams, self.scores):
                self.hyps.add(ids, s, self.prompt_len + len(ids))
        score, ids = sorted(self.hyps.beams, key=lambda x: x[0]).pop()
        if self.prompt_len + len(ids) < self.max_length:
            ids = ids + [self.eos]
        return ids, score


def fork_slots(old, nxt, owned):
    """copy-on-fork slot management of one request's beams.  old: cache slot of each running beam (beam order), nxt: the new
    beams as BeamRequest.process returns them ((score, token, parent beam) in rank order), owned: every slot the request holds.
    A surviving parent keeps its slot for its first child; later children take the slots of beams that died (in `owned`
    order) and must receive the parent's generated rows.  -> (slot of each new beam, [(parent slot, child slot)] forks).
    No slot is both the source and the destination of a fork."""
    kept = {old[p] for _, _, p in nxt}
    free = [s for s in owned if s not in kept]
    new, claimed, forks = [], set(), []
    for _, _, p in nxt:
        if p not in claimed:                    # the parent's first child keeps its slot
            claimed.add(p)
            s = old[p]
        else:                                   # later children fork into the slot of a beam that died
            s = free.pop(0)
            forks.append((old[p], s))
        new.append(s)
    return new, forks
