"""Beam search on the GPU (vsb_beam_candidates_f32 / ops.beam_candidates, vsb_copy_cache_rows_b16 / ops.copy_cache_rows,
VQAEngine.beam_search / generate(num_beams=k)) against oracle/beam_oracle.py.

(1) kernel == oracle triple for triple over k in {1, 2, 4, 16}, R up to 8, both logit dtypes, V in {320, 32000}, with wide
    ties, -inf entries and dominant tokens; a triple may differ only where the oracle's rounding margin is below 1e-6, rarely;
(2) a request's triples do not depend on the other requests of the launch;
(3) the row copy is bit-equal to torch indexing over every layer and refuses a slot that is both a source and a destination;
(4) the engines (bf16, fp16, NF4): num_beams = 1 is greedy; tokens and score == the oracle replayed on the engine's own
    logits; == the fp32 model (oracle/vqa_oracle.py) wherever every decision margin exceeds the engine's logit error;
    generate_batch == one request at a time; the adapter's criteria see [k, len]; free_form_inference(num_beams=3); the
    refusals; device memory back to its level after a beam call."""
import numpy as np
import pytest
import torch

from oracle import beam_oracle as B

pytestmark = pytest.mark.gpu
BF, F16 = torch.bfloat16, torch.float16
MARGIN = 1e-6


def _logits(n_rows, V, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n_rows, V, generator=g) * 3
    x[0] = 0.5                                                            # one row of equal values
    x[1, torch.randperm(V, generator=g)[:int(0.4 * V)]] = -float("inf")
    x[2, int(torch.randint(0, V, (1,), generator=g))] = 60.0              # one dominant token
    if n_rows > 3:
        x[3, : V // 2] = x[3, V // 2:]                                   # every value twice
    return x


def _check(x, rows, scores, k, dtype, got):
    bad = total = 0
    sc, tok, bm = got[0].view(torch.float32).cpu(), got[1].cpu(), got[2].cpu()
    for r in range(rows.shape[0]):
        c = B.candidates(x[rows[r].long()], scores[r].tolist(), k, dtype)
        want = c["cand"]
        mine = list(zip(sc[r].tolist(), tok[r].tolist(), bm[r].tolist()))
        if mine != want:
            assert c["round"] < MARGIN, (r, mine[:4], want[:4], c["round"])
            bad += 1
        total += 1
    return bad, total


@pytest.mark.parametrize("V", [320, 32000])
@pytest.mark.parametrize("dtype", [BF, F16])
def test_candidates_match_oracle(V, dtype):
    from vstar_b200 import ops
    loose = total = 0
    for k in (1, 2, 4, 16):
        for R in (1, 3, 8):
            for k_in in sorted({1, k}):
                n = R * k_in + 5
                x = _logits(n, V, seed=V + 31 * k + R + (dtype == F16))
                g = torch.Generator().manual_seed(k * 100 + R)
                rows = torch.randperm(n, generator=g)[:R * k_in].view(R, k_in).to(torch.int32)
                scores = -(torch.rand(R, k_in, generator=g) * 4).sort(dim=1).values.flip(1) if k_in > 1 else torch.zeros(R, 1)
                if R > 1:
                    scores[1] = -1.25                                     # equal scores: wide ties across beams
                got = ops.beam_candidates(x.cuda(), rows.cuda(), scores.float().cuda(), k, dtype)
                b, t = _check(x, rows, scores.float(), k, dtype, got)
                loose, total = loose + b, total + t
    assert loose <= max(1, total // 50), (loose, total)


def test_candidates_request_independence():
    from vstar_b200 import ops
    V, k = 32000, 4
    x = _logits(40, V, seed=9).cuda()
    g = torch.Generator().manual_seed(2)
    rows = torch.randperm(40, generator=g)[:32].view(8, 4).to(torch.int32).cuda()
    scores = -(torch.rand(8, 4, generator=g) * 3).cuda()
    for dt in (BF, F16):
        full = ops.beam_candidates(x, rows, scores, k, dt)
        for r in (0, 3, 7):
            one = ops.beam_candidates(x, rows[r:r + 1].contiguous(), scores[r:r + 1].contiguous(), k, dt)
            assert torch.equal(one[:, 0], full[:, r])
        perm = torch.tensor([5, 2, 7, 0], device="cuda")
        some = ops.beam_candidates(x, rows[perm].contiguous(), scores[perm].contiguous(), k, dt)
        assert torch.equal(some, full[:, perm])


def test_copy_cache_rows():
    from vstar_b200 import _lib, ops
    L, Bs, T, W = 3, 12, 96, 3 * 256
    cache = torch.randn(L, Bs, T, W, device="cuda").to(BF)
    ref = cache.clone()
    pairs = [(0, 5), (1, 6), (0, 7), (11, 2)]
    ops.copy_cache_rows(cache, pairs, 17, 61)
    for s, d in pairs:
        ref[:, d, 17:61] = ref[:, s, 17:61]
    assert torch.equal(cache.view(torch.int16), ref.view(torch.int16))
    odd = torch.randn(2, 4, 10, 6, device="cuda").to(F16)                # rows that are not 16-byte multiples
    ref = odd.clone()
    ops.copy_cache_rows(odd, [(3, 0)], 0, 10)
    ref[:, 0] = ref[:, 3]
    assert torch.equal(odd.view(torch.int16), ref.view(torch.int16))
    for bad in ([(0, 5), (5, 6)], [(0, 5), (1, 5)], [(0, 12)]):
        with pytest.raises(_lib.VsbError):
            ops.copy_cache_rows(cache, bad, 0, 4)


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
    return cfg, eng, sd, request.param


def _request(cfg, eng, seed):
    rng = np.random.default_rng(seed)
    gen = torch.Generator().manual_seed(seed)
    ids = [1] + rng.integers(3, cfg.vocab - 30, 4 + seed % 5).tolist() + [-200] + rng.integers(3, cfg.vocab - 30, 6 + 3 * seed % 7).tolist()
    img = torch.randn(1, 3, 224, 224, generator=gen)
    return (ids, img.to(eng.dtype).cuda(), None, [seed % 2 == 0], None), img


def _replay(eng, req, k, N, eos, **kw):
    """beam_search with its per-step logits recorded, and the oracle replayed on them"""
    steps = []
    (ids, score), = eng.beam_search([req], k, N, eos, on_step=lambda s, lg, slots, beams: steps.append(
        (lg[slots[0]].float().cpu(), beams[0])), **kw)

    def step_logits(step, beams):
        lg, eb = steps[step]
        assert beams == eb, (step, beams, eb)                             # the oracle walks the engine's path
        return lg
    res = B.beam_search(step_logits, len(req[0]), k, N, eos, eng.dtype, **kw)
    return ids, score, res


def test_num_beams_1_is_greedy(engine):
    cfg, eng, _, _ = engine
    for s in range(3):
        req, _ = _request(cfg, eng, s)
        assert eng.generate(*req, max_new_tokens=8, eos_token_id=-1, num_beams=1) == eng.generate(*req, max_new_tokens=8, eos_token_id=-1)


@pytest.mark.parametrize("k,eos,kw", [(2, -1, {}), (3, 7, dict(length_penalty=0.5)), (4, 11, dict(early_stopping=True)),
                                      (5, 13, dict(early_stopping="never", length_penalty=2.0))])
def test_beam_search_matches_oracle_on_engine_logits(engine, k, eos, kw):
    cfg, eng, _, _ = engine
    for s in range(3):
        req, _ = _request(cfg, eng, s + k)
        ids, score, res = _replay(eng, req, k, 7, eos, **kw)
        assert ids == res["ids"] and score == res["score"], (s, ids, res["ids"], score, res["score"])
        assert eng.generate(*req, max_new_tokens=7, eos_token_id=eos, num_beams=k, **kw) == ids


def test_beam_search_matches_fp32_model(engine):
    """the fp32 reference model (oracle/vqa_oracle.py; for NF4 on the dequantised weights, oracle/nf4_oracle.py) decides like the
    engine wherever every decision margin of the search exceeds the engine's log-prob error (measured on every step of the
    engine's path) plus half a rounding step of the engine dtype, per step.  On this model bf16's rounding step exceeds every decision
    margin, so the cases that must exist are asserted for the fp16 and NF4 engines"""
    from oracle import nf4_oracle, vqa_oracle as V
    cfg, eng, sd, name = engine
    sdf = {n: t.float() for n, t in (nf4_oracle.dequantized_state_dict(sd) if name == "nf4" else sd).items()}
    emb = sdf["model.embed_tokens.weight"]
    agreed = 0
    for s in range(24):
        req, img = _request(cfg, eng, 40 + s)
        k, N = 2 + s % 2, 3
        base = V.build_embeds(sdf, cfg, torch.tensor([req[0]]), img.to(eng.dtype).float(), None, req[3], None)

        @torch.no_grad()
        def step_logits(step, beams):
            rows = []
            for b in beams:
                e = torch.cat([base, emb[torch.tensor(b, dtype=torch.long)].unsqueeze(0)], 1) if b else base
                rows.append(V.forward_logits(sdf, cfg, e)[0, -1].float())
            return torch.stack(rows)
        ref = B.beam_search(step_logits, len(req[0]), k, N, 2, torch.float32)
        steps = []
        (ids, _), = eng.beam_search([req], k, N, 2, on_step=lambda st, lg, slots, beams: steps.append((lg[slots[0]].float().cpu(), beams[0])))
        err = max(float((B.log_probs(lg, torch.float32)[1] - B.log_probs(step_logits(0, b), torch.float32)[1]).abs().max())
                  for lg, b in steps)                                   # on every step of the engine's own path
        tol = N * (err + (2 ** -6 if name == "bf16" else 2 ** -9))          # + half a rounding step at |logp| < 8
        if B.min_margin(ref) > tol:
            assert ids == ref["ids"], (s, ids, ref["ids"], err)
            agreed += 1
    print(f"{name}: {agreed} of 24 searches decided above the tolerance")
    assert agreed >= 1 or name == "bf16"


def test_generate_batch_equals_single(engine):
    cfg, eng, _, _ = engine
    reqs = [_request(cfg, eng, s)[0] for s in (3, 1, 4, 1, 6)]             # lengths differ; requests 1 and 3 are equal
    for k, eos in ((3, 9), (4, -1)):
        batch = eng.beam_search(reqs, k, 6, eos)
        for i, r in enumerate(reqs):
            # the same hypothesis; its score may move in the last bits, since the decode GEMMs of R * k rows and of k rows
            # take different kernels
            (ids, score), = eng.beam_search([r], k, 6, eos)
            assert ids == batch[i][0] and score == pytest.approx(batch[i][1], rel=1e-3), (k, i)
        assert eng.generate_batch(reqs, max_new_tokens=6, eos_token_id=eos, num_beams=k) == [ids for ids, _ in batch]


def test_adapter_and_free_form_inference(engine):
    from PIL import Image
    from vstar_b200.vqa import VQA_LLM, LlavaSearchModel, build_prompt_v1, tokenizer_image_object_token
    cfg, eng, _, _ = engine
    req, img = _request(cfg, eng, 2)
    model = LlavaSearchModel(eng, eos_token_id=-1)
    seen = []

    def criterion(ids, scores):
        seen.append(tuple(ids.shape))
        return ids.shape[1] >= len(req[0]) + 3
    out = model.generate(torch.tensor([req[0]]), images=img, images_long=req[3], num_beams=3, max_new_tokens=8, stopping_criteria=[criterion])
    assert seen == [(3, len(req[0]) + i) for i in (1, 2, 3)]
    best = eng.beam_search([req], 3, 3, -1)[0][0]
    assert out[0, :len(req[0])].tolist() == req[0] and out[0, len(req[0]):].tolist()[:len(best)] == best[:3]
    with pytest.raises(NotImplementedError):
        model.generate(torch.tensor([req[0]]), images=img, do_sample=True, num_beams=2)
    vqa = VQA_LLM(engine=eng)
    pil = Image.fromarray(np.random.default_rng(3).integers(0, 256, (300, 260, 3), dtype=np.uint8), "RGB")
    text = vqa.free_form_inference(pil, "What is on the table?", num_beams=3, max_new_tokens=6)
    ids = tokenizer_image_object_token(build_prompt_v1("<image>\nWhat is on the table?"), vqa.tokenizer)
    pix, _ = vqa._pixels(pil, None)
    new = eng.beam_search([(ids, pix, None, None, None)], 3, 6, vqa.eos)[0][0]
    assert text == vqa.tokenizer.batch_decode([new], skip_special_tokens=True)[0].strip().removesuffix("</s>").strip()
    assert vqa.free_form_inference_batch([pil, pil], ["What is on the table?", "Where?"], max_new_tokens=6, num_beams=3)[0] == text


def test_refusals_and_memory(engine):
    cfg, eng, _, _ = engine
    req, _ = _request(cfg, eng, 1)
    with pytest.raises(NotImplementedError):
        eng.generate(*req, max_new_tokens=4, num_beams=2, temperature=0.7)
    with pytest.raises(ValueError):
        eng.generate(*req, max_new_tokens=4, num_beams=2, stop_ids=[5, 2])
    for k in (0, 17):
        with pytest.raises(ValueError):
            eng.generate(*req, max_new_tokens=4, num_beams=k)
    assert eng.generate(*req, max_new_tokens=4, eos_token_id=2, num_beams=2, stop_ids=[2]) == eng.generate(*req, max_new_tokens=4, num_beams=2)
    eng.generate(*req, max_new_tokens=6, num_beams=4)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    eng.generate(*req, max_new_tokens=6, num_beams=4)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == before
