"""End-to-end parity of the CUDA engine (through the C-ABI) against
  (1) the committed golden vectors produced by the REAL reference (tests/golden, fp32), and
  (2) the CPU oracle run on the same seeded inputs in fp32 and in bf16 (= the reference's bf16 op-by-op rounding).
Tolerance policy (SURVEY.md §8a): the engine computes in bf16 with fp32 accumulation; per stage we require
err_new <= 2 * err_ref + eps where err_ref is the bf16-oracle's error against the fp32 oracle, plus identical
argmax indices / token ids on the golden prompts."""
import json
import os

import numpy as np
import pytest

from tests.helpers import REPORT_DIR
import torch

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(__file__), "golden")
BF = torch.bfloat16
REPORT = {}


def synth_image(seed, w, h):
    from PIL import Image
    return Image.fromarray(np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8), "RGB")


@pytest.fixture(scope="module")
def setup():
    from oracle import vsm_oracle as O
    from vstar_b200.engine import VSMEngine, VSMWeights
    j = json.load(open(os.path.join(G, "tiny_config.json")))
    cfg = O.VSMConfig(**j["cfg"])
    sd = O.synthetic_state_dict(cfg, seed=j["weight_seed"])
    sd_bf = {k: v.to(BF) for k, v in sd.items()}
    eng = VSMEngine(VSMWeights.from_state_dict(cfg, sd), max_tokens=384)
    return O, cfg, sd, sd_bf, eng


def err(a, b):
    a, b = torch.as_tensor(a).float().cpu(), torch.as_tensor(b).float().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def check(name, new, ref_bf16, ref_fp32, floor=4e-3):
    e_new, e_ref = err(new, ref_fp32), err(ref_bf16, ref_fp32)
    REPORT[name] = dict(err_new=e_new, err_ref_bf16=e_ref)
    assert e_new <= 2 * e_ref + floor, (name, e_new, e_ref)


@pytest.mark.parametrize("tag", ["a", "b"])
def test_model_forward_vs_golden_and_oracle(setup, tag):
    O, cfg, sd, sd_bf, eng = setup
    g = np.load(os.path.join(G, f"model_forward_{tag}.npz"))
    w, h = int(g["w"]), int(g["h"])
    img = synth_image(int(g["img_seed"]), w, h)
    ids = torch.from_numpy(g["input_ids"])
    images, images_clip = O.preprocess_owl(img), O.preprocess_clip(img)
    o32 = O.model_forward_inference(sd, cfg, images, images_clip, ids, (h, w))
    o16 = O.model_forward_inference(sd_bf, cfg, images.to(BF), images_clip.to(BF), ids, (h, w))
    out = eng.model_forward(images.to(BF).cuda(), images_clip.to(BF).cuda(), ids.cuda())
    torch.cuda.synchronize()
    r = int(g["loc_row"])
    # golden (reference fp32) == oracle fp32 (pinned on CPU); engine against both
    assert err(o32["hidden"][0, r], g["hidden_loc"]) < 1e-4
    t = f"mf_{tag}_"
    check(t + "hidden_loc", out["hidden_loc"][0], o16["hidden"][0, r], g["hidden_loc"])
    check(t + "seg_query", out["seg_queries"][0], o16["seg_queries"][0], g["seg_query"][0])
    check(t + "det_query", out["det_queries"][0], o16["det_queries"][0], g["det_query"][0])
    gsz = cfg.owl_grid
    fm = out["feature_map"].view(gsz, gsz, -1)[::6, ::6, :]
    check(t + "feature_map", fm, o16["feature_map"][0, ::6, ::6, :], g["fmap_sample"], floor=1e-2)
    check(t + "low_res_mask", out["low_res_masks"][0], o16["low_res_masks"][0, 0], g["low_res_mask"], floor=1e-2)
    check(t + "pred_logits", out["pred_logits"][0], o16["pred_logits"][0, :, 0], g["pred_logits"], floor=1e-2)
    check(t + "pred_boxes", out["pred_boxes"][0], o16["pred_boxes"][0], g["pred_boxes"], floor=1e-2)
    # decision-level parity: same top patch as the fp32 reference, box within 1 px at crop scale
    top_ref = int(np.argmax(g["pred_logits"]))
    top_new = int(out["pred_logits"][0].argmax())
    gap = float(np.sort(g["pred_logits"])[-1] - np.sort(g["pred_logits"])[-2])
    REPORT[t + "top"] = dict(ref=top_ref, new=top_new, top2_gap=gap)
    if gap > 0.05:
        assert top_new == top_ref
    box_px = (out["pred_boxes"][0, top_ref].cpu() - torch.from_numpy(g["pred_boxes"][top_ref])).abs() * torch.tensor([w, h, w, h])
    assert float(box_px.max()) <= 1.0, box_px
    # full-resolution heatmap statistics through the heatmap kernel
    from vstar_b200 import ops
    hm, stats = ops.heatmap(out["low_res_masks"][0].contiguous(), h, w)
    ref_hm = o32["pred_masks"][0].clamp(min=0)
    check(t + "heatmap", hm, o16["pred_masks"][0].float().clamp(min=0), ref_hm, floor=1e-2)


def test_inference_draft_verify_and_generate(setup):
    O, cfg, sd, sd_bf, eng = setup
    g = np.load(os.path.join(G, "generate_a.npz"))
    w, h = int(g["w"]), int(g["h"])
    img = synth_image(int(g["img_seed"]), w, h)
    prompt, forced = torch.from_numpy(g["prompt"]), torch.from_numpy(g["forced"])
    images, images_clip = O.preprocess_owl(img).to(BF).cuda(), O.preprocess_clip(img).to(BF).cuda()
    out = eng.inference(images, images_clip, prompt, forced.tolist(), forced_ids=forced.tolist())
    torch.cuda.synchronize()
    assert out["output_ids"][0].tolist() == g["output_ids"][0].tolist()
    # the greedy argmax at every answer position must equal the reference's step-by-step argmax (golden)
    am = eng.last_argmax[0].tolist()
    REPORT["gen_argmax"] = dict(new=am, ref=g["argmax"].tolist())
    last = torch.from_numpy(g["last_logits"])                       # [steps, V] reference logits per step
    top2 = last.topk(2, dim=-1).values
    for j, (a, b) in enumerate(zip(am, g["argmax"].tolist())):
        if float(top2[j, 0] - top2[j, 1]) > 0.05:
            assert a == b, (j, a, b)
    e = err(eng.last_logits[0].cpu(), last)
    REPORT["gen_logits_err"] = e
    assert e < 3e-2
    check("gen_hidden_loc", out["hidden_loc"][0], torch.from_numpy(g["hidden_loc"]), g["hidden_loc"], floor=2e-2)
    # exact greedy decoding on the KV cache == reference free-running greedy (use_cache=False) on the golden prompt
    ids, argmaxes = eng.generate(prompt, images_clip, max_new_tokens=4, eos_token_id=-1)
    REPORT["gen_free"] = dict(new=argmaxes, ref=g["free_argmax"].tolist())
    assert argmaxes == g["free_argmax"].tolist()


def test_batched_equals_single(setup):
    """frontier batching must not change per-crop results (same kernels, different M)"""
    O, cfg, sd, sd_bf, eng = setup
    prompt, ans = O.synthetic_prompt(cfg, n_text=24, seed=3)
    ids = torch.cat([prompt, ans.unsqueeze(0)], 1)
    imgs = [synth_image(100 + i, 90 + 10 * i, 140 - 7 * i) for i in range(3)]
    ic = torch.cat([O.preprocess_clip(i) for i in imgs]).to(BF).cuda()
    io = torch.cat([O.preprocess_owl(i) for i in imgs]).to(BF).cuda()
    outb = eng.model_forward(io, ic, ids.expand(3, -1).contiguous().cuda())
    lows = outb["low_res_masks"].clone()
    logits = outb["pred_logits"].clone()
    for i in range(3):
        o1 = eng.model_forward(io[i:i + 1], ic[i:i + 1], ids.cuda())
        assert err(lows[i], o1["low_res_masks"][0]) < 2e-2
        assert err(logits[i], o1["pred_logits"][0]) < 2e-2
        assert int(logits[i].argmax()) == int(o1["pred_logits"][0].argmax())


def test_shared_prefix_kv_equals_full_prefill(setup):
    """the K/V rows of the constant text prefix (before <im_start>) are snapshotted by the first prefill and reused by later
    ones, which then run the decoder only from <im_start> on: outputs must equal the full recomputation"""
    O, cfg, sd, sd_bf, eng = setup
    prompt, ans = O.synthetic_prompt(cfg, n_text=40, seed=8)
    ids = torch.cat([prompt, ans.unsqueeze(0)], 1)
    imgs = [synth_image(200 + i, 120 + 20 * i, 100 + 9 * i) for i in range(4)]
    ic = torch.cat([O.preprocess_clip(i) for i in imgs]).to(BF).cuda()
    io = torch.cat([O.preprocess_owl(i) for i in imgs]).to(BF).cuda()
    idb = ids.expand(4, -1).contiguous().cuda()
    keys = ("hidden_loc", "low_res_masks", "pred_logits", "pred_boxes")
    eng.prefix_cache = False
    try:
        full = {k: v.clone() for k, v in eng.model_forward(io, ic, idb).items() if k in keys}
        assert eng._P == 0
    finally:
        eng.prefix_cache = True
    eng._prefix_ids = None                                 # forget whatever an earlier test left behind
    first = {k: v.clone() for k, v in eng.model_forward(io[:2], ic[:2], idb[:2]).items() if k in keys}     # computes + snapshots
    assert eng._P == 0 and eng._prefix_ids is not None
    n0 = eng.stats["prefix_shared"]
    shared = {k: v.clone() for k, v in eng.model_forward(io, ic, idb).items() if k in keys}                # 4 crops, 2 new slots
    img_pos = int((ids[0] == -200).nonzero()[0, 0])
    assert eng._P == img_pos - 1 and eng.stats["prefix_shared"] == n0 + 4
    REPORT["shared_prefix_err"] = {k: err(shared[k], full[k]) for k in keys}
    for k in keys:
        assert torch.equal(first[k], full[k][:2]), k
        # the rows from <im_start> on see bit-identical inputs (same K/V rows, same kernels): EXACT equality, as DESIGN.md states
        assert torch.equal(shared[k], full[k]), (k, err(shared[k], full[k]))
    # draft-verify path on top of the shared prefix
    out = eng.inference(io, ic, prompt.expand(4, -1).contiguous(), ans.tolist(), forced_ids=ans.tolist())
    assert err(out["low_res_masks"], full["low_res_masks"]) < 2e-3 and eng._P == img_pos - 1


def test_prefix_bookkeeping_survives_a_different_prefix_batch(setup):
    """ADVICE r1: a full (P = 0) prefill with ANOTHER prefix overwrites cache rows 0..T of its slots; a later shared-prefix
    prefill must re-copy the snapshot instead of trusting the stale slots"""
    O, cfg, sd, sd_bf, eng = setup
    prompt, ans = O.synthetic_prompt(cfg, n_text=40, seed=8)
    ids = torch.cat([prompt, ans.unsqueeze(0)], 1)
    other = ids.clone()
    other[0, 3] = (int(other[0, 3]) + 7) % 200 + 3            # one different token inside the prefix
    imgs = [synth_image(300 + i, 100 + 10 * i, 90 + 9 * i) for i in range(3)]
    ic = torch.cat([O.preprocess_clip(i) for i in imgs]).to(BF).cuda()
    io = torch.cat([O.preprocess_owl(i) for i in imgs]).to(BF).cuda()
    idb = ids.expand(3, -1).contiguous().cuda()
    keys = ("hidden_loc", "low_res_masks", "pred_logits")
    eng._prefix_ids = None
    want = {k: v.clone() for k, v in eng.model_forward(io, ic, idb).items() if k in keys}          # computes + snapshots
    again = {k: v.clone() for k, v in eng.model_forward(io, ic, idb).items() if k in keys}        # shared prefix
    assert eng._P > 0
    mixed = torch.cat([ids, other], 0).cuda()                 # non-uniform heads: full prefill, snapshot kept
    eng.model_forward(io[:2], ic[:2], mixed)
    assert eng._P == 0 and eng._prefix_slots == 0
    after = {k: v.clone() for k, v in eng.model_forward(io, ic, idb).items() if k in keys}        # must re-copy the prefix rows
    assert eng._P > 0
    for k in keys:
        assert torch.equal(again[k], after[k]), k
        assert err(after[k], want[k]) < 2e-3


def test_cache_grows_instead_of_truncating(setup):
    """ADVICE r1: generation beyond the initial cache rows grows the cache (up to the 2048 RoPE rows); nothing stops silently"""
    O, cfg, sd, sd_bf, eng = setup
    prompt, ans = O.synthetic_prompt(cfg, n_text=24, seed=3)
    img = synth_image(7, 100, 100)
    ic = O.preprocess_clip(img).to(BF).cuda()
    old = eng.max_tokens
    eng.max_tokens, eng._cache, eng._cache_shape = 64, None, None
    try:
        out, am = eng.generate(prompt, ic, max_new_tokens=40, eos_token_id=-1)
        assert len(am) == 40 and eng._cache_shape[2] >= prompt.shape[1] + 255 + 40 - 1
        with pytest.raises(Exception):
            eng._capacity(4096)
    finally:
        eng.max_tokens, eng._cache, eng._cache_shape = old, None, None


def test_zz_write_report(setup):
    os.makedirs(REPORT_DIR, exist_ok=True)
    json.dump(REPORT, open(os.path.join(REPORT_DIR, "engine_parity_report.json"), "w"), indent=1)
    print(json.dumps(REPORT, indent=1))
