"""Sampled decoding on the CPU: the oracle's Philox against Random123's known answers, the oracle's warper chain against
transformers' own TemperatureLogitsWarper / TopKLogitsWarper / TopPLogitsWarper, and the option plumbing of VQA_LLM
(top_p validation, top_k from generation_config.json, seeds from torch's default generator in request order)."""
import json

import numpy as np
import pytest
import torch

from oracle import sampling_oracle as S

BF, F16 = torch.bfloat16, torch.float16


def test_philox_known_answers():
    assert S.philox4x32_10((0, 0, 0, 0), (0, 0)) == (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)
    assert S.philox4x32_10((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2) == (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)
    assert S.philox4x32_10((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0)) == \
        (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)


def test_uniform_depends_on_seed_and_step_only():
    us = [S.uniform(s, t) for s in (0, 1, 2 ** 63 + 5, -7) for t in range(4)]
    assert all(0.0 <= u < 1.0 for u in us) and len(set(us)) == len(us)
    assert S.uniform(-7, 3) == S.uniform(2 ** 64 - 7, 3)                  # the seed is 64 bits, two's complement
    x = S.philox4x32_10((3, 0, 0, 0), (12345, 0))
    assert S.uniform(12345, 3) == ((x[0] >> 5) * 2.0 ** 26 + (x[1] >> 6)) * 2.0 ** -53


def _row(n, seed, dtype, kind):
    """fp32 logits of distinct dtype values in [-12, 4]; `kind` adds a wide tie at the 50th value or -inf entries"""
    g = torch.Generator().manual_seed(seed)
    grid = torch.linspace(-12.0, 4.0, 4000).to(dtype).unique()
    x = grid[torch.randperm(grid.numel(), generator=g)[:n]].float()
    if kind == "tie_k":
        kth = x.sort(descending=True).values[49]
        x[torch.randperm(n, generator=g)[:20]] = kth
    elif kind == "neg_inf":
        x[torch.randperm(n, generator=g)[:n // 4]] = -float("inf")
    return x


def _hf_mask(x, T, top_k, top_p, dtype):
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    s = x.to(dtype).unsqueeze(0)
    if T != 1.0:
        s = TemperatureLogitsWarper(T)(None, s)
        assert torch.equal(s[0].float(), S.scale(x, T, dtype))          # the oracle's rounding and division, bit for bit
    if top_k:
        s = TopKLogitsWarper(top_k)(None, s)
    if top_p is not None and top_p < 1.0:
        s = TopPLogitsWarper(top_p)(None, s.float())                      # the probabilities in fp32
    return (s[0] > -float("inf")).numpy()


def _straddled_group(x, T, top_k, top_p, dtype):
    """bool [n]: the tie group the top-p boundary cuts, if any.  torch.sort is not stable, so HF keeps an arbitrary part of
    it; how many of its tokens survive does not depend on the order (they share one probability)."""
    v = S.scale(x, T, dtype).numpy()
    group = np.zeros(v.size, dtype=bool)
    if top_p is None or top_p >= 1.0:
        return group
    kept = S.sample_row(x, T, top_k, top_p, dtype, 0, 0)["kept"]
    order = S._order(v)
    if len(kept) < len(order) and v[order[len(kept) - 1]] == v[order[len(kept)]]:
        group = v == v[order[len(kept)]]
    return group


@pytest.mark.parametrize("dtype", [F16, BF])
@pytest.mark.parametrize("kind", ["plain", "tie_k", "neg_inf"])
def test_warper_chain_matches_transformers(dtype, kind):
    pytest.importorskip("transformers")
    n = 320
    checked = skipped = 0
    for T in (0.7, 1.0, 1.5):
        for top_k in (0, 1, 50, n):
            for top_p in (None, 0.0, 0.9, 1.0):
                x = _row(n, 0, dtype, kind)
                mask, p_margin = S.warp_mask(x, T, top_k, top_p, dtype)
                mask &= S.scale(x, T, dtype).numpy() > -np.inf
                if p_margin < 1e-6:
                    skipped += 1
                    continue
                hf = _hf_mask(x, T, top_k, top_p, dtype)
                cut = _straddled_group(x, T, top_k, top_p, dtype)
                assert np.array_equal(mask[~cut], hf[~cut]) and mask.sum() == hf.sum(), (T, top_k, top_p)
                checked += 1
                if top_k == 50 and kind == "tie_k" and top_p is None:
                    v = S.scale(x, T, dtype).numpy()
                    assert mask.sum() == (v >= np.sort(v)[::-1][49]).sum() > 50   # every token tied with the 50th value is kept
                if top_p == 0.0:
                    assert mask.sum() == 1
    assert checked >= 45 and skipped <= 2, (checked, skipped)


def test_all_equal_row_keeps_every_token_and_draws_uniformly():
    x = torch.full((320,), 1.25)
    r = S.sample_row(x, 0.7, 50, None, F16, 3, 0)
    assert len(r["kept"]) == 320 and list(r["kept"]) == list(range(320))   # ties in ascending id order
    assert np.allclose(r["probs"], 1 / 320)
    toks = [S.sample_row(x, 0.7, 50, 0.5, F16, 3, t)["token"] for t in range(200)]
    assert max(toks) < 161 and len(set(toks)) > 60                        # top_p = 0.5 keeps the first 160 (+1 at the edge)


def test_inverse_cdf_and_margins():
    x = torch.tensor([2.0, 1.0, 0.0, -1.0, -float("inf")])
    for step in range(50):
        r = S.sample_row(x, 1.0, 0, None, F16, 11, step)
        p = np.exp(np.array([2.0, 1.0, 0.0, -1.0]) - 2.0)
        cdf = np.cumsum(p) / p.sum()
        j = int(np.searchsorted(cdf, r["u"], side="right"))
        assert r["token"] == j and r["u_margin"] == pytest.approx(min(r["u"] - (cdf[j - 1] if j else 0), cdf[j] - r["u"]))
        assert r["token"] != 4


# ------------------------------------------------------------------------------------------------ option plumbing
def test_top_p_validation_and_top_k_argument():
    from vstar_b200.vqa import check_sampling
    assert check_sampling(50, None) == (50, None) and check_sampling(None, 1) == (0, 1.0) and check_sampling(0, 0) == (0, 0.0)
    for bad in (-0.01, 1.5, float("nan")):
        with pytest.raises(ValueError):
            check_sampling(50, bad)
    for bad in (-1, 2.5, True):
        with pytest.raises(ValueError):
            check_sampling(bad, None)


def test_top_k_from_generation_config(tmp_path):
    from vstar_b200.vqa import DEFAULT_TOP_K, generation_top_k
    assert DEFAULT_TOP_K == 50 and generation_top_k(tmp_path) == 50
    (tmp_path / "generation_config.json").write_text(json.dumps({"temperature": 0.9, "top_p": 0.6}))
    assert generation_top_k(tmp_path) == 50
    (tmp_path / "generation_config.json").write_text(json.dumps({"top_k": 7, "max_length": 4096}))
    assert generation_top_k(str(tmp_path)) == 7


class _Tok:
    bos_token_id, eos_token_id = 1, 2

    class _Ids:
        def __init__(self, ids):
            self.input_ids = ids

    def __call__(self, text):
        return self._Ids([1] + [3 + (ord(c) % 50) for c in text])

    def batch_decode(self, seqs, skip_special_tokens=True):
        return ["x" * len(s) for s in seqs]


class _Engine:
    """records the sampling arguments VQA_LLM hands to the engine"""

    class cfg:
        vocab = 320

    dev = "cpu"

    def __init__(self):
        self.calls = []

    def generate(self, *a, **kw):
        self.calls.append(kw)
        return [5, 6]

    def generate_batch(self, reqs, *a, **kw):
        self.calls.append(kw)
        return [[5]] * len(reqs)


def _vqa():
    from vstar_b200.vqa import VQA_LLM
    vqa = VQA_LLM(engine=_Engine(), tokenizer=_Tok())
    vqa._pixels = lambda image, crops: (image, crops)
    return vqa


def test_seeds_come_from_the_default_generator_in_request_order():
    from vstar_b200.vqa import draw_seeds
    vqa = _vqa()
    assert vqa.top_k == 50
    torch.manual_seed(123)
    vqa.free_form_inference_batch([None] * 3, ["a?", "bb?", "c?"], max_new_tokens=4, temperature=0.7, top_p=0.9)
    torch.manual_seed(123)
    want = draw_seeds(3)
    kw = vqa.engine.calls[-1]
    assert kw["seeds"] == want and kw["temperature"] == 0.7 and kw["top_p"] == 0.9 and kw["top_k"] == 50
    torch.manual_seed(123)
    vqa.free_form_inference(None, "a?", temperature=0.7)
    kw = vqa.engine.calls[-1]
    assert kw["seed"] == want[0] and kw["top_p"] is None                 # one draw per request: a single request takes the first
    # greedy decoding draws nothing and passes no sampling
    torch.manual_seed(123)
    vqa.free_form_inference(None, "a?")
    vqa.free_form_inference_batch([None] * 2, ["a?", "b?"], temperature=0)
    assert draw_seeds(1)[0] == want[0]
    assert vqa.engine.calls[-2]["temperature"] == 0 and vqa.engine.calls[-2]["seed"] is None
    assert vqa.engine.calls[-1]["temperature"] == 0 and vqa.engine.calls[-1]["seeds"] is None
    # the reference's warper validation
    for bad in (1.01, -0.5):
        with pytest.raises(ValueError):
            vqa.free_form_inference(None, "a?", temperature=0.7, top_p=bad)
        with pytest.raises(ValueError):
            vqa.free_form_inference_batch([None], ["a?"], temperature=0.7, top_p=bad)
