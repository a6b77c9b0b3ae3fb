"""Sampled decoding on the GPU (vsb_sample_rows_f32 / ops.sample_rows, VQAEngine.generate / generate_batch with temperature > 0)
against oracle/sampling_oracle.py.

(1) kernel == oracle token for token over n in {320, 32000}, T in {0.2, 0.7, 1, 1.5}, top_k in {0, 1, 50, n}, top_p in
    {None, 0, 0.9, 1}, both logit dtypes, with adversarial rows (all equal, a tie at the 50th value wider than the shared-memory
    candidate list, -inf entries, one dominant token); a token may differ only where the oracle's margin is below 1e-6
    (fp32/fp64 summation order), and such rows must be rare;
(2) a row's token does not depend on the other rows of the launch or its position in it;
(3) the drawn tokens follow the oracle's kept-set probabilities (chi-square over 10^5 draws with fixed seeds);
(4) the engines (bf16, fp16, NF4): top_k = 1 == greedy, sampled tokens == the oracle on the logits of the same decode calls
    replayed with those tokens, reproducible seeds, free_form_inference(temperature=0.7) under torch.manual_seed."""
import numpy as np
import pytest
import torch

from oracle import sampling_oracle as S

pytestmark = pytest.mark.gpu
BF, F16 = torch.bfloat16, torch.float16
MARGIN = 1e-6


def _rows(n, B, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, n, generator=g) * 2.5
    x[0] = 1.0                                                            # all equal
    kth = x[1].sort(descending=True).values[49]
    x[1, torch.randperm(n, generator=g)[:max(60, n // 10)]] = kth          # wide tie at the 50th value (> 2048 tokens at n = 32000)
    x[2, torch.randperm(n, generator=g)[:int(0.4 * n)]] = -float("inf")
    x[3, int(torch.randint(0, n, (1,), generator=g))] = 40.0              # one dominant token
    x[4, : n // 2] = x[4, n // 2:]                                        # every value twice
    seeds = torch.randint(-2 ** 63, 2 ** 63 - 1, (B,), generator=g, dtype=torch.int64)
    return x, seeds


@pytest.mark.parametrize("n", [320, 32000])
@pytest.mark.parametrize("dtype", [BF, F16])
def test_kernel_matches_oracle(n, dtype):
    from vstar_b200 import ops
    B = 64
    x, seeds = _rows(n, B, seed=n + (dtype == F16))
    xd, sd = x.cuda(), seeds.cuda()
    total = loose = 0
    for T in (0.2, 0.7, 1.0, 1.5):
        for top_k in (0, 1, 50, n):
            for top_p in (None, 0.0, 0.9, 1.0):
                step = 3 + top_k % 7
                got = ops.sample_rows(xd, T, top_k, top_p, dtype, sd, step)
                for Bs in (1, 3):                                         # smaller launches give the same tokens
                    assert torch.equal(ops.sample_rows(xd[:Bs], T, top_k, top_p, dtype, sd[:Bs], step), got[:Bs])
                got = got.cpu().numpy()
                want, margin = S.sample_rows(x, T, top_k, top_p, dtype, seeds.tolist(), step)
                bad = got != want
                assert not (bad & (margin >= MARGIN)).any(), \
                    (T, top_k, top_p, np.nonzero(bad)[0][:5], got[bad][:5], want[bad][:5], margin[bad][:5])
                loose += int(bad.sum())
                total += B
    assert loose <= max(2, total // 1000), (loose, total)


def test_row_independence():
    """the same rows in another order and among other rows: every row keeps its token"""
    from vstar_b200 import ops
    x, seeds = _rows(32000, 40, seed=5)
    y, sy = _rows(32000, 24, seed=6)
    perm = torch.randperm(40, generator=torch.Generator().manual_seed(1))
    for T, k, p in ((0.7, 50, 0.9), (1.0, 0, 0.9), (1.5, 50, None)):
        for dt in (BF, F16):
            a = ops.sample_rows(x.cuda(), T, k, p, dt, seeds.cuda(), 11)
            mixed = torch.cat([y[:7], x[perm], y[7:]]).cuda()
            ms = torch.cat([sy[:7], seeds[perm], sy[7:]]).cuda()
            b = ops.sample_rows(mixed, T, k, p, dt, ms, 11)
            assert torch.equal(b[7:47], a[perm.cuda()])
            for i in (0, 13, 39):
                assert torch.equal(ops.sample_rows(x[i:i + 1].cuda(), T, k, p, dt, seeds[i:i + 1].cuda(), 11), a[i:i + 1])


def test_bad_arguments_raise():
    from vstar_b200 import _lib, ops
    x, s = torch.zeros(2, 320, device="cuda"), torch.zeros(2, dtype=torch.int64, device="cuda")
    for kw in (dict(temperature=0.0), dict(top_p=1.5), dict(top_p=-0.1), dict(top_k=-1)):
        a = dict(temperature=0.7, top_k=50, top_p=None)
        a.update(kw)
        with pytest.raises(_lib.VsbError):
            ops.sample_rows(x, a["temperature"], a["top_k"], a["top_p"], BF, s, 0)


@pytest.mark.parametrize("n,T,top_k,top_p", [(320, 0.7, 50, 0.9), (32000, 1.0, 0, 0.9), (32000, 1.5, 50, None), (320, 1.0, 0, None)])
def test_distribution(n, T, top_k, top_p):
    """10^5 draws (1000 copies of one row with their own seeds x 100 steps) against the oracle's renormalised kept-set
    probabilities: no token outside the kept set, chi-square p-value > 1e-4 (fixed seeds: deterministic)"""
    from scipy import stats
    from vstar_b200 import ops
    g = torch.Generator().manual_seed(n + top_k)
    row = torch.randn(n, generator=g) * 1.5
    R, steps = 1000, 100
    xd = row.cuda().expand(R, n).contiguous()
    seeds = torch.randint(-2 ** 63, 2 ** 63 - 1, (R,), generator=g, dtype=torch.int64).cuda()
    toks = torch.cat([ops.sample_rows(xd, T, top_k, top_p, BF, seeds, s) for s in range(steps)]).cpu().numpy()
    r = S.sample_row(row, T, top_k, top_p, BF, 0, 0)
    kept, probs = r["kept"], r["probs"]
    pos = np.full(n, -1)
    pos[kept] = np.arange(len(kept))
    assert (pos[toks] >= 0).all()
    counts = np.bincount(pos[toks], minlength=len(kept)).astype(np.float64)
    exp = probs * len(toks)
    big = exp >= 5                                                        # pool the rare tokens into one cell
    obs_c = np.append(counts[big], counts[~big].sum())
    exp_c = np.append(exp[big], exp[~big].sum())
    if exp_c[-1] < 5:
        obs_c, exp_c = obs_c[:-1], exp_c[:-1]
        obs_c[-1] += counts[~big].sum()
        exp_c[-1] += exp[~big].sum()
    pval = stats.chisquare(obs_c, exp_c * obs_c.sum() / exp_c.sum()).pvalue
    assert pval > 1e-4, (pval, len(kept))


# ------------------------------------------------------------------------------------------------ engines
@pytest.fixture(scope="module", params=["bf16", "fp16", "nf4"])
def engine(request):
    from oracle import vqa_oracle as V, vsm_oracle as O
    from vstar_b200 import synth
    from vstar_b200.vqa import VQAEngine, VQAWeights
    cfg = O.tiny_config()
    sd = {k: synth.synthetic_tensor(k, shp, seed=4321) for k, shp in V.vqa_state_dict_shapes(cfg).items()}
    kw = dict(bf16=dict(), fp16=dict(dtype=F16), nf4=dict(dtype=F16, quant="nf4"))[request.param]
    eng = VQAEngine(VQAWeights.from_state_dict(cfg, sd, **kw), max_tokens=1024)
    return cfg, eng


def _request(cfg, eng, seed):
    rng = np.random.default_rng(seed)
    gen = torch.Generator().manual_seed(seed)
    ids = [1] + rng.integers(3, cfg.vocab - 30, 4 + seed % 5).tolist() + [-200] + rng.integers(3, cfg.vocab - 30, 6 + 3 * seed % 7).tolist()
    return (ids, torch.randn(1, 3, 224, 224, generator=gen).to(eng.dtype).cuda(), None, [seed % 2 == 0], None)


def _replay_single(eng, req, out, max_new_tokens):
    """the logits generate() saw at every step, recomputed by the same calls with the emitted tokens"""
    ids, img, crops, il, ol = req
    x = eng.build_embeds(ids, img, crops, il, ol)
    T = x.shape[0]
    eng.prefill_embeds(x, reserve=max(0, min(max_new_tokens, eng.MAX_POSITIONS - T)))
    rows = [eng.last_logits(x)[0].cpu()]
    for s, t in enumerate(out[:-1]):
        rows.append(eng.append_tokens([t], T + s)[0].cpu())
    return rows


def _check_tokens(rows, out, T, top_k, top_p, dtype, seed):
    for step, (lg, t) in enumerate(zip(rows, out)):
        r = S.sample_row(lg, T, top_k, top_p, dtype, seed, step)
        assert r["token"] == t or r["margin"] < MARGIN, (step, r["token"], t, r["margin"])
        if r["token"] != t:
            return                                                        # paths part at a rounding-level tie


def test_engine_top_k_1_is_greedy(engine):
    cfg, eng = engine
    for s in range(3):
        req = _request(cfg, eng, s)
        greedy = eng.generate(*req, max_new_tokens=8, eos_token_id=-1)
        sampled = eng.generate(*req, max_new_tokens=8, eos_token_id=-1, temperature=0.7, top_k=1, top_p=0.9, seed=1234 + s)
        if sampled != greedy:
            # only where the fp32 argmax and a token tied with it after rounding to the engine dtype part ways
            rows = _replay_single(eng, req, greedy, 8)
            j = next(i for i in range(8) if sampled[i] != greedy[i])
            v = S.scale(rows[j], 0.7, eng.dtype)
            assert v[sampled[j]] == v[greedy[j]] == v.max(), (s, j)


def test_engine_sampled_generate_matches_oracle(engine):
    cfg, eng = engine
    for s, (T, k, p) in enumerate([(0.7, 50, None), (1.0, 50, 0.9), (1.5, 0, 0.9), (0.2, 0, None)]):
        req = _request(cfg, eng, s)
        seed = 99 + 7 * s
        out = eng.generate(*req, max_new_tokens=8, eos_token_id=-1, temperature=T, top_k=k, top_p=p, seed=seed)
        assert len(out) == 8
        assert eng.generate(*req, max_new_tokens=8, eos_token_id=-1, temperature=T, top_k=k, top_p=p, seed=seed) == out
        _check_tokens(_replay_single(eng, req, out, 8), out, T, k, p, eng.dtype, seed)


def test_engine_sampled_generate_batch_matches_oracle(engine):
    cfg, eng = engine
    reqs = [_request(cfg, eng, s) for s in (3, 1, 4, 1)]                   # lengths differ; requests 1 and 3 are equal
    seeds = [5, -6, 2 ** 62 + 7, 11]
    T, k, p, N = 1.0, 50, 0.9, 6
    outs = eng.generate_batch(reqs, max_new_tokens=N, eos_token_id=-1, temperature=T, top_k=k, top_p=p, seeds=seeds)
    assert eng.generate_batch(reqs, max_new_tokens=N, eos_token_id=-1, temperature=T, top_k=k, top_p=p, seeds=seeds) == outs
    # replay: the same ordering by length as generate_batch, the same ragged calls with the emitted tokens
    xs = eng.build_embeds_batch(reqs)
    perm = sorted(range(len(xs)), key=lambda i: int(xs[i].shape[0]))
    xs = [xs[i] for i in perm]
    longest = max(int(x.shape[0]) for x in xs)
    logits, Tpad, lens = eng.prefill_ragged(xs, reserve=max(0, min(N, eng.MAX_POSITIONS - longest)))
    rows = [logits.cpu()]
    for step in range(N - 1):
        rows.append(eng.decode_ragged([outs[i][step] for i in perm], lens, Tpad, step).cpu())
    for b, i in enumerate(perm):
        _check_tokens([r[b] for r in rows], outs[i], T, k, p, eng.dtype, seeds[i])


def test_free_form_inference_sampled_is_reproducible(engine):
    from PIL import Image
    from vstar_b200.vqa import VQA_LLM
    cfg, eng = engine
    vqa = VQA_LLM(engine=eng)
    img = Image.fromarray(np.random.default_rng(3).integers(0, 256, (300, 260, 3), dtype=np.uint8), "RGB")
    texts = []
    for _ in range(2):
        torch.manual_seed(17)
        texts.append(vqa.free_form_inference(img, "What is on the table?", temperature=0.7, max_new_tokens=6))
        texts.append(tuple(vqa.free_form_inference_batch([img, img], ["What is it?", "Where?"], max_new_tokens=6, temperature=0.7,
                                                         top_p=0.9)))
    assert texts[0] == texts[2] and texts[1] == texts[3]
    with pytest.raises(ValueError):
        vqa.free_form_inference(img, "q", temperature=0.7, top_p=2.0)
