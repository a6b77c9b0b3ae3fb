"""Beam-search semantics (oracle/beam_oracle.py, vstar_b200/beam.py) on the CPU.

(1) the oracle == the installed transformers' generate(num_beams=k, length_penalty=0) on tiny fp32 Llamas (at lp = 0 lengths
    drop out, so 4.31's and the installed version's rules agree), k in {2, 3, 4}, with an eos bias that ends some hypotheses;
    compared where every decision margin exceeds the fp32-vs-fp64 log-softmax difference;
(2) hand-built score tables pin the rules specific to transformers 4.31;
(3) k = 1 is greedy decoding; the host scorer the engine runs equals the oracle on random candidate tables;
(4) length_penalty / early_stopping come from generation_config.json."""
import json
import math

import numpy as np
import pytest
import torch

from oracle import beam_oracle as B

F32 = torch.float32
EOS = 2


def _tiny_llama(seed, eos_bias):
    from transformers import LlamaConfig, LlamaForCausalLM
    torch.manual_seed(seed)
    cfg = LlamaConfig(vocab_size=64, hidden_size=32, intermediate_size=64, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=4, max_position_embeddings=128, initializer_range=0.3, bos_token_id=1, eos_token_id=EOS,
                      pad_token_id=0)
    model = LlamaForCausalLM(cfg).eval()
    bias = torch.zeros(64)
    bias[EOS] = eos_bias
    model.lm_head.register_forward_hook(lambda m, i, o: o + bias)
    return model


def _callback(model, prompt):
    @torch.no_grad()
    def step_logits(step, beams):
        ids = torch.tensor([prompt + b for b in beams])
        return model(input_ids=ids).logits[:, -1].float()
    return step_logits


@pytest.mark.parametrize("k", [2, 3, 4])
def test_oracle_matches_transformers_at_lp0(k):
    compared = by_eos = by_len = 0
    for seed in range(8):
        model = _tiny_llama(seed, eos_bias=(0.0, 1.0, 2.0, 3.0)[seed % 4])
        prompt = [1] + torch.randint(3, 64, (5 + seed % 3,), generator=torch.Generator().manual_seed(seed)).tolist()
        N = 6 + seed % 3
        res = B.beam_search(_callback(model, prompt), len(prompt), k, N, EOS, F32, length_penalty=0.0)
        if B.min_margin(res) < 1e-4:                                   # fp32 (torch) against fp64 (oracle) log-softmax
            continue
        with torch.no_grad():
            out = model.generate(torch.tensor([prompt]), num_beams=k, do_sample=False, max_new_tokens=N, length_penalty=0.0,
                                 early_stopping=False, eos_token_id=EOS, pad_token_id=0, num_return_sequences=1,
                                 return_dict_in_generate=True, output_scores=True)
        got = out.sequences[0, len(prompt):].tolist()
        assert got == res["ids"], (seed, got, res["ids"])
        assert out.sequences_scores[0].item() == pytest.approx(res["score"], abs=1e-4)
        compared += 1
        by_eos += len(res["hyp"]) < N
        by_len += len(res["hyp"]) == N
    assert compared >= 4 and by_eos >= 1 and by_len >= 1, (compared, by_eos, by_len)


def test_k1_is_greedy():
    for seed in range(4):
        model = _tiny_llama(seed, eos_bias=2.0 * (seed % 2))
        prompt = [1, 7, 9, 11, 13]
        res = B.beam_search(_callback(model, prompt), len(prompt), 1, 8, EOS, F32)
        with torch.no_grad():
            g = model.generate(torch.tensor([prompt]), do_sample=False, num_beams=1, max_new_tokens=8, eos_token_id=EOS, pad_token_id=0)
        assert g[0, len(prompt):].tolist() == res["ids"]


# ------------------------------------------------------------------------------------------------ hand-built tables
def _table(rows, V=8):
    """rows: per beam {token: log-prob} (the rest -inf); logits = those log-probs (log_softmax leaves a normalised row as is)"""
    x = torch.full((len(rows), V), -float("inf"))
    for i, r in enumerate(rows):
        for t, v in r.items():
            x[i, t] = math.log(v)
    return x


def _run(tables, prompt_len, k, N, **kw):
    return B.beam_search(lambda step, beams: tables[step][:len(beams)], prompt_len, k, N, EOS, F32, **kw)


def test_prompt_counted_in_length_and_eos_appended():
    # step 0: eos is the best candidate (rank 0 < k): a hypothesis with no generated ids, length = the prompt's ids
    # (ids [1, 5, -200, 7]: the <image> placeholder counts once, the spliced rows not at all)
    t0 = _table([{EOS: 0.5, 3: 0.3, 4: 0.2}])
    t1 = _table([{5: 0.1, 6: 0.9}, {5: 0.1, 6: 0.9}])
    prompt = [1, 5, -200, 7]
    res = _run([t0, t1, t1], len(prompt), 2, 3, length_penalty=1.0)
    assert res["hyp"] == [] and res["ids"] == [EOS]                        # eos excluded from the hypothesis, appended on output
    assert res["score"] == pytest.approx(float(torch.tensor(math.log(0.5), dtype=F32)) / 4, rel=1e-6)
    # with the prompt left out (the installed transformers' rule) the length would be 0 and the score undefined: pinned above


def test_eos_at_rank_k_or_worse_is_skipped():
    t0 = _table([{3: 0.4, 4: 0.35, EOS: 0.25}])                            # eos at rank 2 = k: skipped
    res = _run([t0], 3, 2, 1)
    assert res["hyp"] == [3]
    assert len(res["margins"]["insert"]) == 2                              # only the two open beams, at finalize


def test_early_stopping_modes():
    # step 0: beams [3] (log .6) and [4] (log .4); step 1: eos is the best token of both (ranks 0, 1) -> two hypotheses of
    # length 5, worst = (log .4 + log .8) / 5 = -0.228; the running beams go on at -2.53 / -2.81 and lose log .99 per step
    t0 = _table([{3: 0.6, 4: 0.4}])
    t1 = _table([{EOS: 0.9, 5: 0.1}, {EOS: 0.8, 6: 0.2}])
    t2 = _table([{5: 0.99, 6: 0.01}, {5: 0.99, 6: 0.01}])
    prompt_len, N = 4, 12
    steps = {}
    for es in (True, False, "never"):
        res = _run([t0, t1] + [t2] * (N - 2), prompt_len, 2, N, early_stopping=es, length_penalty=1.0)
        steps[es] = len(res["history"])
        assert res["hyp"] == [3]                                           # the eos hypothesis of beam [3]
    # True: done once k hypotheses exist (step 1).  False: at step 2, best = log .4 + log .2 + log .99 = -2.536 and
    # -0.228 >= -2.536 / cur_len 6.  "never": -2.536 / max_length 16 = -0.158 > -0.228, and so on to max_new_tokens
    assert steps == {True: 2, False: 3, "never": N}


def test_finalize_tie_goes_to_the_later_entry():
    # two open beams with equal scores and equal lengths: the later one in the list (rank 1) is returned
    t0 = _table([{3: 0.5, 4: 0.5}])
    res = _run([t0], 3, 2, 1)
    assert res["hyp"] == [4] and res["margins"]["pick"] == 0.0
    h = B.Hypotheses(2, 1.0, False, 10)
    h.add([7], -1.0, 2)
    h.add([8], -1.0, 2)
    assert sorted(h.beams, key=lambda x: x[0]).pop()[1] == [8]


def test_host_scorer_equals_oracle_on_random_tables():
    from vstar_b200.beam import BeamRequest
    rng = np.random.default_rng(0)
    for trial in range(60):
        k = int(rng.integers(1, 6))
        V = 12
        N = int(rng.integers(1, 7))
        lp = float(rng.choice([0.0, 1.0, 2.0, -0.5]))
        es = [True, False, "never"][trial % 3]
        tables = []
        for step in range(N):
            x = torch.tensor(rng.normal(size=(k if step else 1, V)) * 2, dtype=F32)
            x[:, EOS] += float(rng.choice([0.0, 2.0]))
            tables.append(x)
        res = B.beam_search(lambda s, beams: tables[s][:len(beams)], 5, k, N, EOS, F32, length_penalty=lp, early_stopping=es)
        q = BeamRequest(k, 5, N, EOS, lp, es)
        for step in range(N):
            c = B.candidates(tables[step][:len(q.beams)], q.scores, k, F32)["cand"]
            q.process(c)
            if q.done or step == N - 1:
                break
        ids, score = q.finalize()
        assert ids == res["ids"] and score == res["score"], trial


def test_defaults_from_generation_config(tmp_path):
    from vstar_b200.vqa import generation_top_k
    assert generation_top_k(tmp_path, beams=True) == (50, 1.0, False)
    (tmp_path / "generation_config.json").write_text(json.dumps({"top_k": 20, "length_penalty": 0.5, "early_stopping": "never"}))
    assert generation_top_k(tmp_path, beams=True) == (20, 0.5, "never")
    assert generation_top_k(tmp_path) == 20
    (tmp_path / "generation_config.json").write_text(json.dumps({"early_stopping": True}))
    assert generation_top_k(tmp_path, beams=True) == (50, 1.0, True)


def test_bad_beam_arguments():
    from vstar_b200.beam import check_beams
    for k in (0, 17, 2.0, True):
        with pytest.raises(ValueError):
            check_beams(k, False)
    with pytest.raises(ValueError):
        check_beams(2, "sometimes")
