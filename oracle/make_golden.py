"""TEST INFRASTRUCTURE ONLY — generates tests/golden/*.npz from the REAL reference.

Run where a checkout of the reference is available (oracle/ref_shims.py, VSTAR_REFERENCE_ROOT):

    python -m oracle.make_golden

What it does
  1. imports the reference's own VSMForCausalLM / visual_search (read-only,
     through oracle/ref_shims.py) at the tiny golden config,
  2. loads the deterministic synthetic weights (oracle.vsm_oracle.synthetic_state_dict)
     into it,
  3. runs the reference on seeded inputs and writes its outputs as golden
     vectors,
  4. asserts the CPU restatement (oracle/vsm_oracle.py) reproduces every one of
     them (fp32: rtol 1e-4 / atol 1e-5; ids / argmax / trajectories identical).

The goldens are what pins the oracle wherever the reference is not available
(every test run).
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_shims, vsm_oracle as O  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def hf_cfgs(cfg: O.VSMConfig):
    owl = dict(
        vision_config=dict(hidden_size=cfg.owl_hidden, intermediate_size=cfg.owl_inter,
                           num_hidden_layers=cfg.owl_layers, num_attention_heads=cfg.owl_heads,
                           image_size=cfg.owl_image, patch_size=cfg.owl_patch, hidden_act="quick_gelu",
                           layer_norm_eps=cfg.vit_eps),
        text_config=dict(hidden_size=cfg.owl_query_dim, intermediate_size=128, num_hidden_layers=1,
                         num_attention_heads=2, vocab_size=64, max_position_embeddings=16),
        projection_dim=64)
    clip = dict(hidden_size=cfg.clip_hidden, intermediate_size=cfg.clip_inter, num_hidden_layers=cfg.clip_layers,
                num_attention_heads=cfg.clip_heads, image_size=cfg.clip_image, patch_size=cfg.clip_patch,
                layer_norm_eps=cfg.vit_eps, hidden_act="quick_gelu", projection_dim=64)
    return owl, clip


def build_reference_model(cfg: O.VSMConfig, sd):
    owl, clip = hf_cfgs(cfg)
    ref_shims.install(owl, clip)
    from VisualSearch.model.VSM import VSMForCausalLM
    from VisualSearch.model.llava.model.language_model.llava_llama import LlavaConfig
    lc = LlavaConfig(hidden_size=cfg.hidden, intermediate_size=cfg.intermediate, num_hidden_layers=cfg.n_layers,
                     num_attention_heads=cfg.n_heads, num_key_value_heads=cfg.n_heads, vocab_size=cfg.vocab,
                     rms_norm_eps=cfg.rms_eps, max_position_embeddings=2048, train_mask_decoder=True,
                     out_dim=cfg.owl_query_dim, mm_vision_select_layer=cfg.clip_select_layer,
                     mm_use_im_start_end=True, vision_tower="fake-clip", mm_vision_tower="fake-clip",
                     mm_hidden_size=cfg.clip_hidden, attn_implementation="eager")
    torch.manual_seed(0)
    m = VSMForCausalLM(lc, loc_token_idx=cfg.loc_token_idx, is_eval=True)
    m.get_model().initialize_vision_modules(m.get_model().config)
    m.eval()
    ref_keys = set(m.state_dict().keys())
    missing_in_ref = [k for k in sd if k not in ref_keys]
    assert not missing_in_ref, missing_in_ref
    m.load_state_dict(sd, strict=False)
    return m


def synth_image(seed, w, h):
    from PIL import Image
    arr = np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)
    return Image.fromarray(arr, "RGB")


def ref_model_forward(m, images, images_clip, ids, size):
    L = ids.shape[1]
    with torch.no_grad():
        return m.model_forward(images=images, images_clip=images_clip, input_ids=ids, labels=None,
                               attention_masks=torch.ones(1, L, dtype=torch.long), offset=torch.tensor([0, 1]),
                               masks_list=[None], label_list=[torch.zeros(*size)], bboxes_labels_list=[None],
                               bboxes_valid_list=None, masks_valid_list=None, resize_list=[(768, 768)],
                               inference=True)


def close(a, b, name, rtol=1e-4, atol=2e-5):
    a, b = torch.as_tensor(a).float(), torch.as_tensor(b).float()
    err = (a - b).abs().max().item()
    ok = torch.allclose(a, b, rtol=rtol, atol=atol)
    print(f"  {name:28s} max|d|={err:.3e} ref|max|={b.abs().max().item():.3e} {'OK' if ok else 'MISMATCH'}")
    assert ok, name


def case_model_forward(m, sd, cfg, tag, img_seed, w, h, n_text):
    print(f"[golden] model_forward case {tag}")
    img = synth_image(img_seed, w, h)
    images_clip = O.preprocess_clip(img)
    images = O.preprocess_owl(img)
    prompt, ans = O.synthetic_prompt(cfg, n_text=n_text, seed=img_seed)
    ids = torch.cat([prompt, ans.unsqueeze(0)], dim=1)
    ref = ref_model_forward(m, images, images_clip, ids, (h, w))
    with torch.no_grad():
        ref_lm = super(type(m), m).forward(images=images_clip, attention_mask=torch.ones_like(ids), input_ids=ids,
                                            output_hidden_states=True)
        ref_fmap = m.get_visual_embs(images)
    orc = O.model_forward_inference(sd, cfg, images, images_clip, ids, (h, w))
    close(orc["hidden"], ref_lm.hidden_states, "hidden")
    close(orc["logits"], ref_lm.logits, "logits", atol=1e-4)
    close(orc["feature_map"], ref_fmap, "owl feature_map")
    close(orc["pred_masks"][0], ref["pred_masks"][0][0], "pred_mask", atol=1e-4)
    close(orc["pred_logits"], ref["pred_logits"], "pred_logits", atol=1e-4)
    close(orc["pred_boxes"], ref["pred_boxes"], "pred_boxes")
    loc_row = int((ids[0] == cfg.loc_token_idx).nonzero()[0, 0]) - 1 + 255
    pm = ref["pred_masks"][0][0]
    g = dict(
        img_seed=img_seed, w=w, h=h, input_ids=ids.numpy(),
        loc_row=loc_row,
        hidden_loc=ref_lm.hidden_states[0, loc_row].numpy(),
        hidden_last=ref_lm.hidden_states[0, -1].numpy(),
        logits_argmax=ref_lm.logits[0].argmax(-1).numpy(),
        logits_last=ref_lm.logits[0, -1].numpy(),
        fmap_sample=ref_fmap[0, ::6, ::6, :].numpy(),
        seg_query=orc["seg_queries"].numpy(),     # oracle value (verified == reference downstream)
        det_query=orc["det_queries"].numpy(),
        low_res_mask=orc["low_res_masks"][0, 0].numpy(),
        pred_mask_stats=np.array([pm.max().item(), pm.min().item(), pm.clamp(min=0).sum().item(),
                                  float(pm.argmax())], dtype=np.float64),
        pred_mask_sample=pm[::7, ::7].numpy(),
        pred_logits=ref["pred_logits"][0, :, 0].numpy(),
        pred_boxes=ref["pred_boxes"][0].numpy(),
    )
    np.savez_compressed(os.path.join(GOLDEN_DIR, f"model_forward_{tag}.npz"), **g)


def case_generate(m, sd, cfg, tag, img_seed, w, h, n_text):
    """Greedy loop restated around the REFERENCE forward (HF generate of the
    reference's VSMForCausalLM.inference does not run under transformers 5.5,
    SURVEY.md §8c)."""
    print(f"[golden] generate case {tag}")
    img = synth_image(img_seed, w, h)
    images_clip = O.preprocess_clip(img)
    prompt, ans = O.synthetic_prompt(cfg, n_text=n_text, seed=img_seed)
    ids = prompt.clone()
    ref_argmax, ref_last_logits = [], []
    for step in range(len(ans)):
        with torch.no_grad():
            out = super(type(m), m).forward(images=images_clip, attention_mask=torch.ones_like(ids), input_ids=ids,
                                             output_hidden_states=True)
        ref_argmax.append(int(out.logits[0, -1].argmax()))
        ref_last_logits.append(out.logits[0, -1].numpy().copy())
        ids = torch.cat([ids, ans[step].view(1, 1)], dim=1)
        if int(ans[step]) == 2:
            break
    o_ids, o_hidden, o_argmax = O.greedy_generate(sd, cfg, prompt, images_clip, max_new_tokens=100, eos_token_id=2,
                                                  forced_ids=ans)
    assert o_argmax == ref_argmax, (o_argmax, ref_argmax)
    assert torch.equal(o_ids, ids)
    close(o_hidden, out.hidden_states, "last-step hidden")
    # free-running (unforced) greedy for a few tokens too
    ids2 = prompt.clone()
    free = []
    for step in range(4):
        with torch.no_grad():
            out2 = super(type(m), m).forward(images=images_clip, attention_mask=torch.ones_like(ids2), input_ids=ids2)
        t = int(out2.logits[0, -1].argmax())
        free.append(t)
        ids2 = torch.cat([ids2, torch.tensor([[t]])], dim=1)
    o2_ids, _, o2_argmax = O.greedy_generate(sd, cfg, prompt, images_clip, max_new_tokens=4, eos_token_id=-1)
    assert o2_argmax == free, (o2_argmax, free)
    np.savez_compressed(os.path.join(GOLDEN_DIR, f"generate_{tag}.npz"), img_seed=img_seed, w=w, h=h,
                        prompt=prompt.numpy(), forced=ans.numpy(), argmax=np.array(ref_argmax),
                        last_logits=np.stack(ref_last_logits), free_argmax=np.array(free),
                        output_ids=ids.numpy(), hidden_loc=out.hidden_states[0, -3].numpy())


# ---------------------------------------------------------------- search goldens
from tests.helpers import FakeNLP, StubVSM  # noqa: E402  (deterministic stub VSM + rule parser standing in for spaCy)


def trajectory(search_path):
    return np.array([st["bbox"] for st in search_path], dtype=np.int64)


def case_search(tag, img_seed, w, h, smallest, hot=None, **kw):
    print(f"[golden] search case {tag}")
    import visual_search as RVS  # the reference module
    from vstar_b200.noun_chunks import extract_noun_chunks
    nlp = FakeNLP()
    RVS.nlp = nlp                # the reference's module-level spaCy pipeline (visual_search.py:10) -> deterministic rule parser
    img = synth_image(img_seed, w, h)
    stub = StubVSM(hot)
    fs, pl, ok, av = RVS.visual_search(stub, img, "mug", None, smallest, **kw)
    ref_calls = list(stub.calls)
    stub2 = StubVSM(hot)
    fs2, pl2, ok2, av2, path2 = O.visual_search(stub2, img, "mug", None, smallest,
                                                extract_noun_chunks=lambda t: extract_noun_chunks(t, nlp), **kw)
    assert ref_calls == stub2.calls
    assert pl == pl2 and ok == ok2 and fs["bbox"] == fs2["bbox"]
    assert torch.equal(fs["detection_result"], fs2["detection_result"])
    assert (av is None) == (av2 is None) and (av is None or torch.equal(av, av2))
    cues = [st.get("context_cue", "") for st in path2]
    np.savez_compressed(os.path.join(GOLDEN_DIR, f"search_{tag}.npz"), img_seed=img_seed, w=w, h=h, smallest=smallest,
                        kw=json.dumps(kw), hot=str(hot), all_valid_boxes=(av.numpy() if av is not None else np.zeros((0, 4), np.float32)),
                        has_all_valid=int(av is not None), calls=np.array(ref_calls, dtype=np.int64).reshape(-1, 3),
                        trajectory=trajectory(path2), path_length=pl, success=int(ok), final_bbox=np.array(fs["bbox"]),
                        detection_result=fs["detection_result"].numpy(), context_cues=json.dumps(cues))
    n_one = sum(1 for c in cues if c and not c.split("#")[-1].startswith("region "))
    print(f"   {len(ref_calls)} VSM calls, path_length={pl}, success={ok}, weak-cue nodes={sum(1 for c in cues if c)} "
          f"(single-chunk phrases: {n_one})")


class RefModelVSM:
    """visual_search.VSM-shaped wrapper around the REFERENCE model graph with
    teacher-forced ids (no tokenizer offline): used to pin an end-to-end
    trajectory produced by reference search loop x reference model."""

    def __init__(self, m, cfg):
        self.m, self.cfg = m, cfg
        prompt, ans = O.synthetic_prompt(cfg, n_text=24, seed=5)
        self.ids = torch.cat([prompt, ans.unsqueeze(0)], dim=1)
        self.calls = 0

    def inference(self, image, question, mode="segmentation"):
        self.calls += 1
        images_clip = O.preprocess_clip(image)
        images = O.preprocess_owl(image)
        out = ref_model_forward(self.m, images, images_clip, self.ids, (image.height, image.width))
        pm = torch.clamp(out["pred_masks"][0], min=0)[-1]
        if mode == "segmentation":
            return pm
        return out["pred_boxes"][0], out["pred_logits"][0].sigmoid(), pm


class OracleVSM:
    def __init__(self, sd, cfg):
        self.sd, self.cfg = sd, cfg
        prompt, ans = O.synthetic_prompt(cfg, n_text=24, seed=5)
        self.ids = torch.cat([prompt, ans.unsqueeze(0)], dim=1)

    def inference(self, image, question, mode="segmentation"):
        out = O.model_forward_inference(self.sd, self.cfg, O.preprocess_owl(image), O.preprocess_clip(image), self.ids,
                                        (image.height, image.width))
        pm = torch.clamp(out["pred_masks"], min=0)[-1]
        if mode == "segmentation":
            return pm
        return out["pred_boxes"][0], out["pred_logits"][0].sigmoid(), pm


def case_search_model(m, sd, cfg, tag, img_seed, w, h, smallest, **kw):
    print(f"[golden] search+model case {tag}")
    import visual_search as RVS
    img = synth_image(img_seed, w, h)
    with torch.no_grad():
        fs, pl, ok, av = RVS.visual_search(RefModelVSM(m, cfg), img, "mug", None, smallest, **kw)
        fs2, pl2, ok2, av2, path2 = O.visual_search(OracleVSM(sd, cfg), img, "mug", None, smallest, **kw)
    assert pl == pl2 and ok == ok2 and fs["bbox"] == fs2["bbox"], (pl, pl2, fs["bbox"], fs2["bbox"])
    close(fs2["detection_result"], fs["detection_result"], "final detection_result", atol=1e-2)
    np.savez_compressed(os.path.join(GOLDEN_DIR, f"search_model_{tag}.npz"), img_seed=img_seed, w=w, h=h,
                        smallest=smallest, kw=json.dumps(kw), trajectory=trajectory(path2), path_length=pl,
                        success=int(ok), final_bbox=np.array(fs["bbox"]),
                        detection_result=fs["detection_result"].numpy(),
                        scores=np.array([st["score"] if st["score"] is not None else np.nan for st in path2], dtype=np.float64))
    print(f"   path_length={pl}, success={ok}, nodes={len(path2)}")


def search_model_separated(m, sd, cfg):
    """BASELINE configs[1]-shaped searches (root + 4 crops, depth 2) whose four child priorities are separated by 1.3e-2 ... 2e-2
    (seeds picked by scanning 40 images with the oracle): far more than the bf16 score error, so the product must reproduce the
    reference's expansion order EXACTLY on these (the 21-node cases above always contain near-ties below 1e-3)."""
    for tag, seed in (("d", 99), ("e", 87)):
        case_search_model(m, sd, cfg, tag, img_seed=seed, w=640, h=512, smallest=300, confidence_high=2.0,
                          target_cue_threshold=-1e9, target_cue_threshold_minimum=-1e9)


def build_reference_vqa_model(cfg, sd):
    owl, clip = hf_cfgs(cfg)
    ref_shims.install(owl, clip)
    from LLaVA.llava.model.language_model.llava_search_llama import LlavaSearchLlamaForCausalLM, LlavaSearchConfig
    lc = LlavaSearchConfig(hidden_size=cfg.hidden, intermediate_size=cfg.intermediate, num_hidden_layers=cfg.n_layers,
                           num_attention_heads=cfg.n_heads, num_key_value_heads=cfg.n_heads, vocab_size=cfg.vocab,
                           rms_norm_eps=cfg.rms_eps, max_position_embeddings=2048, mm_vision_tower="openai/fake-clip",
                           mm_hidden_size=cfg.clip_hidden, mm_vision_select_layer=cfg.clip_select_layer,
                           mm_projector_type="linear", object_mm_projector_type="perceiver", mm_use_im_start_end=False,
                           attn_implementation="eager")
    torch.manual_seed(0)
    m = LlavaSearchLlamaForCausalLM(lc)
    m.get_model().get_vision_tower().load_model()
    m.eval()
    ref_keys = set(m.state_dict().keys())
    assert all(k in ref_keys for k in sd), [k for k in sd if k not in ref_keys][:5]
    missing = m.load_state_dict(sd, strict=False)
    assert not [k for k in missing.missing_keys if "post_layernorm" not in k and "position_ids" not in k], missing.missing_keys[:5]
    return m


def case_vqa(tag, img_seed):
    """SEAL VQA-LLM forward (image short + 2 object crops long, the k<=2 configuration of vstar_bench_eval.py:231-236),
    option scoring and a short greedy generation, from the REAL reference LlavaSearchLlamaForCausalLM."""
    from oracle import vqa_oracle as V
    from vstar_b200 import synth
    print(f"[golden] vqa case {tag}")
    cfg = O.tiny_config()
    shapes = V.vqa_state_dict_shapes(cfg)
    sd = {k: synth.synthetic_tensor(k, shp, seed=4321) for k, shp in shapes.items()}
    m = build_reference_vqa_model(cfg, sd)
    g = torch.Generator().manual_seed(img_seed)
    image = torch.randn(1, 3, 224, 224, generator=g)
    crops = torch.randn(2, 3, 224, 224, generator=g)
    hi = cfg.vocab - 24
    q = torch.randint(3, hi, (1, 30), generator=g)
    q[0, 0] = 1
    q[0, 6] = -200
    q[0, 20] = -300
    q[0, 24] = -300
    opts = [torch.randint(3, hi, (n,), generator=g) for n in (3, 5, 4, 2)]
    for images_long, objects_long, sub in (([False], [True, True], "short_long"), ([True], [False, False], "long_short")):
        with torch.no_grad():
            ref = m(q, images=image, object_features=crops, images_long=images_long, objects_long=objects_long).logits
        emb = V.build_embeds(sd, cfg, q, image, crops, images_long, objects_long)
        orc = V.forward_logits(sd, cfg, emb)
        close(orc, ref, f"vqa logits {sub}", atol=1e-4)
        # option losses through full teacher-forced forwards of the reference (== its shared-prefix KV reuse)
        ref_losses = []
        for o in opts:
            full = torch.cat([q, o.unsqueeze(0)], dim=1)
            with torch.no_grad():
                lg = m(full, images=image, object_features=crops, images_long=images_long, objects_long=objects_long).logits
            Tq = ref.shape[1]
            ref_losses.append(torch.nn.functional.cross_entropy(lg[0, Tq - 1:Tq - 1 + o.numel()], o))
        ref_losses = torch.stack(ref_losses)
        o_losses, o_choice = V.option_losses(sd, cfg, q, opts, image, crops, images_long, objects_long)
        close(o_losses, ref_losses, f"option NLL {sub}", atol=1e-4)
        assert o_choice == int(ref_losses.argmin())
        # greedy generation around the reference forward
        ids = q.clone()
        gen = []
        for _ in range(4):
            with torch.no_grad():
                lg = m(ids, images=image, object_features=crops, images_long=images_long, objects_long=objects_long).logits
            t = int(lg[0, -1].argmax())
            gen.append(t)
            ids = torch.cat([ids, torch.tensor([[t]])], dim=1)
        assert V.free_form_generate(sd, cfg, q, image, crops, images_long, objects_long, max_new_tokens=4, eos_token_id=-1) == gen
        np.savez_compressed(os.path.join(GOLDEN_DIR, f"vqa_{tag}_{sub}.npz"), img_seed=img_seed, q=q.numpy(),
                            opts=np.concatenate([o.numpy() for o in opts]), opt_lens=np.array([o.numel() for o in opts]),
                            images_long=np.array(images_long), objects_long=np.array(objects_long),
                            logits_last=ref[0, -1].numpy(), logits_argmax=ref[0].argmax(-1).numpy(), T=ref.shape[1],
                            option_losses=ref_losses.numpy(), gen=np.array(gen))


def case_bench_eval():
    """the reference's own eval_model (vstar_bench_eval.py:168-273) over a tiny synthetic benchmark tree, with the stub VQA /
    stub VSM injected in place of the two model classes; its output JSON is the golden for vstar_b200.bench_eval."""
    print("[golden] bench_eval")
    import tempfile
    import types
    import vstar_bench_eval as E   # the reference module
    from tests.helpers import StubVQA, make_bench_folder
    with tempfile.TemporaryDirectory() as tmp:
        folder = make_bench_folder(os.path.join(tmp, "bench"))
        out = os.path.join(tmp, "out.json")
        E.VQA_LLM = lambda args: StubVQA()
        E.VSM = lambda args: StubVSM()
        E.eval_model(types.SimpleNamespace(benchmark_folder=folder, output_path=out, vsm_model_path="stub", minimum_size_scale=4.0,
                                           minimum_size=224))
        res = json.load(open(out))
    for t in res:
        res[t] = sorted(res[t], key=lambda r: r["image"])       # os.listdir order is file-system dependent
    with open(os.path.join(GOLDEN_DIR, "bench_eval_golden.json"), "w") as f:
        json.dump(res, f, indent=1)
    print("   ", {t: len(v) for t, v in res.items()}, "samples;", sum(len(r["search_result"]) for v in res.values() for r in v), "search results")


def search_edge_cases():
    """termination / selection branches of visual_search() (visual_search.py:399-413, :428-431, :497-512)"""
    case_search("edge_root_hit", img_seed=24, w=1280, h=960, smallest=224, hot="root")          # success at the root, 3 valid boxes
    case_search("edge_deep_hit", img_seed=25, w=1100, h=1000, smallest=224, hot="small")        # success below the root
    case_search("edge_tiny", img_seed=26, w=200, h=150, smallest=224)                           # root is already the smallest unit
    case_search("edge_tiny_unsure", img_seed=26, w=200, h=150, smallest=224, confidence_low=0.9)  # nothing passes confidence_low
    case_search("edge_wide", img_seed=27, w=2000, h=420, smallest=224, confidence_high=2.0)      # 4x1 splits (h/w <= 0.5)
    case_search("edge_odd", img_seed=28, w=1001, h=777, smallest=251, confidence_high=2.0)       # sizes not divisible by the grid


def case_host_logic():
    """results of the reference's host functions on the inputs of the drivers in tests/test_host_logic_vs_reference.py"""
    import visual_search as RVS
    import vstar_bench_eval as E
    from LLaVA.llava import conversation as rc_vqa
    from LLaVA.llava.mm_utils import tokenizer_image_object_token as ref_tok_obj
    from VisualSearch.model.llava import conversation as rc_vsm
    from VisualSearch.model.llava.mm_utils import tokenizer_image_token as ref_tok
    from VisualSearch.utils.utils import expand2square as ref_e2s_vsm

    from tests import test_host_logic_vs_reference as H
    from tests.helpers import FakeNLP, NumpyScorer  # noqa: F401
    from vstar_b200 import vsm
    from vstar_b200.config import tiny_config
    nlp = FakeNLP()
    RVS.nlp = nlp
    tok = vsm.SyntheticTokenizer(tiny_config())
    prompts = []
    for q in H.QUESTIONS:
        conv = rc_vsm.conv_templates["llava_v1"].copy()
        conv.append_message(conv.roles[0], ("<image>" + "\n" + q).replace("<image>", "<im_start><image><im_end>"))
        conv.append_message(conv.roles[1], "")
        llama2 = []
        for use_se in (True, False):                 # the other template the CLI accepts (visual_search.py:48)
            c2 = rc_vsm.conv_templates["llava_llama_2"].copy()
            c2.messages = []
            p2 = "<image>" + "\n" + q
            if use_se:
                p2 = p2.replace("<image>", "<im_start><image><im_end>")
            c2.append_message(c2.roles[0], p2)
            c2.append_message(c2.roles[1], "")
            llama2.append(c2.get_prompt())
        vqa_cases = []
        for answer in (None, "the mug is red"):      # SEAL VQA LLM (vstar_bench_eval.py:79-85, :112-116, :136-139)
            cv = rc_vqa.conv_templates["v1"].copy()
            qs = "<image>" + "\n" + "Additional visual information to focus on: mug <object> at location [0.1,0.2,0.3,0.4]; dog <object>.\n" + q
            cv.append_message(cv.roles[0], qs)
            cv.append_message(cv.roles[1], answer)
            vqa_cases.append([cv.get_prompt(), ref_tok_obj(cv.get_prompt(), tok, -200, return_tensors="pt").tolist()])
        prompts.append(dict(vsm_v1=conv.get_prompt(), vsm_llama_2=llama2, vsm_ids=ref_tok(conv.get_prompt(), tok, return_tensors="pt").tolist(),
                            vqa=vqa_cases))
    gold = dict(
        split_and_sub_patches=H.run_split_and_sub_patches(RVS.split_4subpatches, RVS.get_sub_patches),
        refine_bbox_and_iou=H.run_refine_bbox_and_iou(RVS.refine_bbox, RVS.iou),
        prioritize_pop_order=H.run_prioritize_pop_order(RVS.Prioritize),
        prompts_and_token_splicing=prompts,
        padding_and_patch_geometry=H.run_padding_and_patch_geometry(ref_e2s_vsm, E.expand2square, E.VQA_LLM.get_patch),
        noun_chunks=H.run_noun_chunks(RVS.extract_noun_chunks, RVS.get_noun_chunks, RVS.tranverse, RVS.filter_chunk_list, nlp),
        visualisation_files=H.run_visualisation_files(RVS.visual_search),
    )
    with open(H.GOLD, "w") as f:
        json.dump(H.blockwise(gold), f, separators=(",", ":"))


def main():
    if os.environ.get("GOLDEN_ONLY") == "host_logic":
        assert ref_shims.reference_available()
        ref_shims.install(*hf_cfgs(O.tiny_config()))
        return case_host_logic()
    if os.environ.get("GOLDEN_ONLY") == "search_edges":
        assert ref_shims.reference_available()
        ref_shims.install(*hf_cfgs(O.tiny_config()))
        return search_edge_cases()
    if os.environ.get("GOLDEN_ONLY") == "search_model_separated":
        assert ref_shims.reference_available()
        torch.set_num_threads(8)
        cfg = O.tiny_config()
        sd = O.synthetic_state_dict(cfg, seed=1234)
        return search_model_separated(build_reference_model(cfg, sd), sd, cfg)
    if os.environ.get("GOLDEN_ONLY") == "bench_eval":
        assert ref_shims.reference_available()
        ref_shims.install(*hf_cfgs(O.tiny_config()))
        return case_bench_eval()
    assert ref_shims.reference_available(), "needs a checkout of the reference (VSTAR_REFERENCE_ROOT)"
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    torch.set_num_threads(8)
    cfg = O.tiny_config()
    sd = O.synthetic_state_dict(cfg, seed=1234)
    m = build_reference_model(cfg, sd)
    with open(os.path.join(GOLDEN_DIR, "tiny_config.json"), "w") as f:
        json.dump(dict(cfg=cfg.to_dict(), weight_seed=1234), f, indent=1)
    case_model_forward(m, sd, cfg, "a", img_seed=11, w=150, h=110, n_text=24)
    case_model_forward(m, sd, cfg, "b", img_seed=12, w=96, h=233, n_text=60)
    case_generate(m, sd, cfg, "a", img_seed=13, w=128, h=128, n_text=24)
    case_search("stub_3lvl", img_seed=21, w=1024, h=1024, smallest=224, confidence_high=2.0)
    case_search("stub_default", img_seed=22, w=1500, h=700, smallest=224)
    case_search("stub_weakcue", img_seed=23, w=900, h=1900, smallest=300, confidence_high=2.0,
                target_cue_threshold=50.0, target_cue_threshold_minimum=40.0)
    # strong and weak cues mixed (threshold inside the stub's score range): both branches of visual_search.py:422-443, and
    # phrases with zero / one / several noun chunks
    case_search("stub_mixcue", img_seed=29, w=1600, h=1200, smallest=224, confidence_high=2.0,
                target_cue_threshold=9.5, target_cue_threshold_minimum=9.5)
    search_edge_cases()
    case_search_model(m, sd, cfg, "a", img_seed=31, w=640, h=512, smallest=200, confidence_high=2.0,
                      target_cue_threshold=-1e9, target_cue_threshold_minimum=-1e9)
    # more reference-model x reference-search trajectories: another seed, and a tall image whose root splits 1x4
    case_search_model(m, sd, cfg, "b", img_seed=32, w=600, h=600, smallest=160, confidence_high=2.0,
                      target_cue_threshold=-1e9, target_cue_threshold_minimum=-1e9)
    case_search_model(m, sd, cfg, "c", img_seed=33, w=300, h=960, smallest=200, confidence_high=2.0,
                      target_cue_threshold=-1e9, target_cue_threshold_minimum=-1e9)
    search_model_separated(m, sd, cfg)
    case_vqa("a", img_seed=41)
    case_bench_eval()
    case_host_logic()
    print("golden vectors written to", GOLDEN_DIR)


if __name__ == "__main__":
    main()
