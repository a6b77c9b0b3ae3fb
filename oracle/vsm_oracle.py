"""TEST INFRASTRUCTURE ONLY — CPU restatement (oracle) of the V* VSM hot path.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline /
`--impl reference` leg may import this module, and only as the checker / the
reported CPU baseline.  The product (`vstar_b200/`) never imports it.

Parity pin status: the reference (penghao-wu/vstar @ 4ede664) ships NO tests,
golden vectors or fixtures (SURVEY.md §4) -> "parity unpinned" by the
reference's own tests.  Instead this restatement is pinned against OUTPUTS OF
THE REFERENCE ITSELF: `oracle/make_golden.py` imports the reference's own
`VSMForCausalLM.model_forward(inference=True)` / `LlavaLlamaForCausalLM.forward`
/ `visual_search()` (read-only, via `oracle/ref_shims.py`) in the build
container, runs them on seeded random-init weights, and commits the results as
`tests/golden/*.npz`; `tests/test_oracle_golden.py` checks this file against
those vectors (and, when the reference is available, against the live
reference).

The restatement is written with plain torch ops in the dtype of the weights it
is given: fp32 weights give the fp32 oracle; bf16 weights reproduce the
reference's bf16 op-by-op rounding (used to bound `err_new <= 2*err_ref`).

State-dict key layout = the reference model's own `state_dict()` (which is
also the checkpoint layout written by
/root/reference/VisualSearch/merge_lora_weights_and_save_hf_model.py:143-151).

Third-party arithmetic restated here (not part of the reference): HF
transformers `LlamaModel`, `CLIPVisionModel`, `OwlViTForObjectDetection` heads
(reference pins transformers==4.31.0, requirements.txt:43); citations below use
the installed 5.5.0 source paths `transformers/models/...` as in SURVEY.md §8a.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field, asdict
from queue import PriorityQueue
import functools

import numpy as np
import torch
import torch.nn.functional as F

from vstar_b200.config import VSMConfig, tiny_config, IMAGE_TOKEN_INDEX  # noqa: E402,F401  (architecture description only)
from vstar_b200.synth import (state_dict_shapes, synthetic_state_dict, synthetic_tensor,  # noqa: E402,F401
                              synthetic_prompt)


# --------------------------------------------------------------------------
# small helpers
# --------------------------------------------------------------------------
def _lin(sd, name, x):
    b = sd.get(name + ".bias")
    return F.linear(x, sd[name + ".weight"], b)


def _ln(sd, name, x, eps):
    return F.layer_norm(x, (x.shape[-1],), sd[name + ".weight"], sd[name + ".bias"], eps)


def quick_gelu(x):
    # transformers/activations.py:117-123  x * sigmoid(1.702 x)
    return x * torch.sigmoid(1.702 * x)


# --------------------------------------------------------------------------
# ViT encoder shared by CLIP-L/14 and OWL-ViT-B/16
#   transformers/models/clip/modeling_clip.py:146-158 (embeddings), :261-279,
#   :291-329 (attention), :339-382 (layer), :659-677 (pre_layrnorm);
#   transformers/models/owlvit/modeling_owlvit.py:274-293, :742-782
# --------------------------------------------------------------------------
def vit_embed(sd, p, pixel, patch):
    w = sd[p + "embeddings.patch_embedding.weight"]
    x = F.conv2d(pixel.to(w.dtype), w, None, stride=patch)          # [B,C,g,g]
    x = x.flatten(2).transpose(1, 2)                                 # [B,g*g,C]
    cls = sd[p + "embeddings.class_embedding"].expand(x.shape[0], 1, -1)
    x = torch.cat([cls, x], dim=1)
    return x + sd[p + "embeddings.position_embedding.weight"].unsqueeze(0)


def vit_layer(sd, p, x, heads, eps):
    B, S, C = x.shape
    hd = C // heads
    h = _ln(sd, p + "layer_norm1", x, eps)
    q = _lin(sd, p + "self_attn.q_proj", h).view(B, S, heads, hd).transpose(1, 2)
    k = _lin(sd, p + "self_attn.k_proj", h).view(B, S, heads, hd).transpose(1, 2)
    v = _lin(sd, p + "self_attn.v_proj", h).view(B, S, heads, hd).transpose(1, 2)
    att = torch.matmul(q, k.transpose(-1, -2)) * (hd ** -0.5)
    att = torch.softmax(att, dim=-1, dtype=torch.float32).to(q.dtype)
    o = torch.matmul(att, v).transpose(1, 2).reshape(B, S, C)
    x = x + _lin(sd, p + "self_attn.out_proj", o)
    h = _ln(sd, p + "layer_norm2", x, eps)
    h = _lin(sd, p + "mlp.fc2", quick_gelu(_lin(sd, p + "mlp.fc1", h)))
    return x + h


def clip_features(sd, cfg: VSMConfig, images_clip):
    """CLIPVisionTower.forward + feature_select
    (/root/reference/VisualSearch/model/llava/model/multimodal_encoder/clip_encoder.py:31-60):
    hidden_states[select_layer][:, 1:].  hidden_states[i] = output of layer i-1
    (index 0 = after pre_layrnorm), so select_layer=-2 needs layers 0..L-2."""
    p = "model.vision_tower.vision_tower.vision_model."
    x = vit_embed(sd, p, images_clip, cfg.clip_patch)
    x = _ln(sd, p + "pre_layrnorm", x, cfg.vit_eps)
    n_run = cfg.clip_layers + 1 + cfg.clip_select_layer if cfg.clip_select_layer < 0 else cfg.clip_select_layer
    for i in range(n_run):
        x = vit_layer(sd, f"{p}encoder.layers.{i}.", x, cfg.clip_heads, cfg.vit_eps)
    return x[:, 1:]


def encode_images(sd, cfg, images_clip):
    # /root/reference/VisualSearch/model/llava/model/llava_arch.py:93-96
    return _lin(sd, "model.mm_projector", clip_features(sd, cfg, images_clip))


def owl_visual_embs(sd, cfg: VSMConfig, images):
    """OwlViT.get_visual_embs (/root/reference/VisualSearch/model/owlvit/owlvit.py:121-148)."""
    p = "model.owlvit.vision_model."
    x = vit_embed(sd, p, images, cfg.owl_patch)
    x = _ln(sd, p + "pre_layernorm", x, cfg.vit_eps)
    for i in range(cfg.owl_layers):
        x = vit_layer(sd, f"{p}encoder.layers.{i}.", x, cfg.owl_heads, cfg.vit_eps)
    x = _ln(sd, p + "post_layernorm", x, cfg.vit_eps)
    x = x[:, 1:, :] * x[:, :1, :]
    x = _ln(sd, "model.owlvit.layer_norm", x, cfg.vit_eps)
    g = cfg.owl_grid
    return x.reshape(x.shape[0], g, g, x.shape[-1])


# --------------------------------------------------------------------------
# Llama (transformers/models/llama/modeling_llama.py:53-67 RMSNorm, :117-168
# RoPE, :171-184 MLP, :199-221 eager attention)
# --------------------------------------------------------------------------
def rmsnorm(x, w, eps):
    dt = x.dtype
    xf = x.to(torch.float32)
    xf = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
    return w * xf.to(dt)


def rope_cos_sin(T, hd, theta, dtype, start=0):
    inv = 1.0 / (theta ** (torch.arange(0, hd, 2, dtype=torch.float32) / hd))
    pos = torch.arange(start, start + T, dtype=torch.float32)
    fr = torch.outer(pos, inv)
    emb = torch.cat([fr, fr], dim=-1)
    return emb.cos().to(dtype), emb.sin().to(dtype)


def rotate_half(x):
    h = x.shape[-1] // 2
    return torch.cat([-x[..., h:], x[..., :h]], dim=-1)


def llama_forward(sd, cfg: VSMConfig, embeds):
    """Full-sequence causal forward (use_cache=False semantics,
    /root/reference/VisualSearch/model/VSM.py:151).  Returns the final-normed
    last-layer states [B,T,d] (what the reference exposes as `hidden_states`
    in eval, llava_llama.py:124-135)."""
    B, T, d = embeds.shape
    H, hd = cfg.n_heads, cfg.head_dim
    cos, sin = rope_cos_sin(T, hd, cfg.rope_theta, embeds.dtype)
    cos, sin = cos.to(embeds.device), sin.to(embeds.device)
    mask = torch.full((T, T), float("-inf"), dtype=embeds.dtype, device=embeds.device).triu(1)
    x = embeds
    for i in range(cfg.n_layers):
        p = f"model.layers.{i}."
        h = rmsnorm(x, sd[p + "input_layernorm.weight"], cfg.rms_eps)
        q = F.linear(h, sd[p + "self_attn.q_proj.weight"]).view(B, T, H, hd).transpose(1, 2)
        k = F.linear(h, sd[p + "self_attn.k_proj.weight"]).view(B, T, H, hd).transpose(1, 2)
        v = F.linear(h, sd[p + "self_attn.v_proj.weight"]).view(B, T, H, hd).transpose(1, 2)
        q = q * cos + rotate_half(q) * sin
        k = k * cos + rotate_half(k) * sin
        att = torch.matmul(q, k.transpose(2, 3)) * (hd ** -0.5) + mask
        att = torch.softmax(att, dim=-1, dtype=torch.float32).to(q.dtype)
        o = torch.matmul(att, v).transpose(1, 2).reshape(B, T, d)
        x = x + F.linear(o, sd[p + "self_attn.o_proj.weight"])
        h = rmsnorm(x, sd[p + "post_attention_layernorm.weight"], cfg.rms_eps)
        g = F.silu(F.linear(h, sd[p + "mlp.gate_proj.weight"])) * F.linear(h, sd[p + "mlp.up_proj.weight"])
        x = x + F.linear(g, sd[p + "mlp.down_proj.weight"])
    return rmsnorm(x, sd["model.norm.weight"], cfg.rms_eps)


def splice_embeds(sd, cfg, input_ids_1d, image_feats):
    """prepare_inputs_labels_for_multimodal, mm_use_im_start_end branch
    (/root/reference/VisualSearch/model/llava/model/llava_arch.py:185-208,
    :235-256): the single -200 placeholder is replaced by the 256 projected
    image rows; everything else is an embed_tokens lookup."""
    emb = sd["model.embed_tokens.weight"]
    pos = (input_ids_1d == IMAGE_TOKEN_INDEX).nonzero()
    assert pos.numel() == 1, "exactly one image placeholder expected"
    p = int(pos[0, 0])
    return torch.cat([emb[input_ids_1d[:p]], image_feats.to(emb.dtype), emb[input_ids_1d[p + 1:]]], dim=0)


def lm_forward(sd, cfg, input_ids, images_clip, image_feats=None):
    """LlavaLlamaForCausalLM.forward (llava_llama.py:55-135): -> (logits [B,T,V], hidden [B,T,d])."""
    if image_feats is None:
        image_feats = encode_images(sd, cfg, images_clip)
    embeds = torch.stack([splice_embeds(sd, cfg, input_ids[b], image_feats[b]) for b in range(input_ids.shape[0])])
    hidden = llama_forward(sd, cfg, embeds)
    logits = F.linear(hidden, sd["lm_head.weight"])
    return logits, hidden


def greedy_generate(sd, cfg, input_ids, images_clip, max_new_tokens=100, eos_token_id=2, forced_ids=None):
    """Restated HF greedy `generate` with use_cache=False
    (/root/reference/VisualSearch/model/VSM.py:451-458; llava_llama.py:137-163:
    past_key_values=None -> the full ids AND the image are re-run each step).
    `forced_ids` emulates the logits-processor used for synthetic weights
    (SURVEY.md §8d) — the same forcing is applied to the CUDA path.
    Returns (output_ids [1,L], last-step hidden [1,L-1+255,d], per-step argmax list)."""
    assert input_ids.shape[0] == 1
    ids = input_ids.clone()
    argmaxes = []
    hidden = None
    for step in range(max_new_tokens):
        logits, hidden = lm_forward(sd, cfg, ids, images_clip)
        nxt = int(torch.argmax(logits[0, -1].float()))
        argmaxes.append(nxt)
        if forced_ids is not None and step < len(forced_ids):
            nxt = int(forced_ids[step])
        ids = torch.cat([ids, torch.tensor([[nxt]], dtype=ids.dtype, device=ids.device)], dim=1)
        if nxt == eos_token_id:
            break
    return ids, hidden, argmaxes


# --------------------------------------------------------------------------
# [LOC] row selection + query MLPs  (VSM.py:465-490 / :222-234, :282-297)
# --------------------------------------------------------------------------
def loc_mask_from_output_ids(output_ids, loc_idx):
    m = output_ids[:, 1:] == loc_idx
    return torch.cat([torch.zeros((m.shape[0], 255), dtype=torch.bool, device=m.device), m], dim=1)


def text_fcs(sd, which, hidden):
    p = f"model.text_hidden_fcs_{which}.0."
    return _lin(sd, p + "2", F.relu(_lin(sd, p + "0", hidden)))


# --------------------------------------------------------------------------
# SAM prompt encoder / two-way transformer / mask decoder
#   /root/reference/VisualSearch/model/segment_anything/modeling/
#   prompt_encoder.py:140-186,:189-229; transformer.py:62-106,:151-182,:220-242;
#   mask_decoder.py:15-27,:138-186; common.py:31-43
# --------------------------------------------------------------------------
def dense_pe(sd, g):
    G = sd["model.prompt_encoder.pe_layer.positional_encoding_gaussian_matrix"]
    grid = torch.ones((g, g), dtype=G.dtype, device=G.device)
    y = (grid.cumsum(dim=0) - 0.5) / g
    x = (grid.cumsum(dim=1) - 0.5) / g
    c = torch.stack([x, y], dim=-1)
    c = 2 * c - 1
    c = c @ G
    c = 2 * np.pi * c
    pe = torch.cat([torch.sin(c), torch.cos(c)], dim=-1)
    return pe.permute(2, 0, 1).unsqueeze(0)          # [1,256,g,g]


def sam_attention(sd, p, q, k, v, heads):
    q = _lin(sd, p + "q_proj", q)
    k = _lin(sd, p + "k_proj", k)
    v = _lin(sd, p + "v_proj", v)
    b, n, c = q.shape
    sep = lambda t: t.reshape(t.shape[0], t.shape[1], heads, t.shape[2] // heads).transpose(1, 2)
    q, k, v = sep(q), sep(k), sep(v)
    cph = q.shape[-1]
    att = q @ k.permute(0, 1, 3, 2)
    att = att / math.sqrt(cph)
    att = torch.softmax(att, dim=-1)              # NOTE: activation dtype, no fp32 upcast
    o = att @ v
    o = o.transpose(1, 2).reshape(b, o.shape[2], heads * cph)
    return _lin(sd, p + "out_proj", o)


def two_way_transformer(sd, cfg, src, pos_src, tokens):
    p = "model.mask_decoder.transformer."
    bs, c, h, w = src.shape
    keys = src.flatten(2).permute(0, 2, 1)
    key_pe = pos_src.flatten(2).permute(0, 2, 1)
    queries = tokens
    query_pe = tokens
    H = cfg.sam_heads
    for i in range(cfg.sam_depth):
        lp = f"{p}layers.{i}."
        if i == 0:
            queries = sam_attention(sd, lp + "self_attn.", queries, queries, queries, H)
        else:
            q = queries + query_pe
            queries = queries + sam_attention(sd, lp + "self_attn.", q, q, queries, H)
        queries = _ln(sd, lp + "norm1", queries, 1e-5)
        q = queries + query_pe
        k = keys + key_pe
        queries = queries + sam_attention(sd, lp + "cross_attn_token_to_image.", q, k, keys, H)
        queries = _ln(sd, lp + "norm2", queries, 1e-5)
        mlp = _lin(sd, lp + "mlp.lin2", F.relu(_lin(sd, lp + "mlp.lin1", queries)))
        queries = _ln(sd, lp + "norm3", queries + mlp, 1e-5)
        q = queries + query_pe
        k = keys + key_pe
        keys = keys + sam_attention(sd, lp + "cross_attn_image_to_token.", k, q, queries, H)
        keys = _ln(sd, lp + "norm4", keys, 1e-5)
    q = queries + query_pe
    k = keys + key_pe
    queries = queries + sam_attention(sd, p + "final_attn_token_to_image.", q, k, keys, H)
    queries = _ln(sd, p + "norm_final_attn", queries, 1e-5)
    return queries, keys


def layernorm2d(x, w, b, eps=1e-6):
    u = x.mean(1, keepdim=True)
    s = (x - u).pow(2).mean(1, keepdim=True)
    x = (x - u) / torch.sqrt(s + eps)
    return w[:, None, None] * x + b[:, None, None]


def sam_upsample(sd, p, x):
    # mask_decoder.py:24-27 : bilinear x2 in fp32, cast back, conv3x3 pad 1
    x = F.interpolate(x.float(), scale_factor=2.0, mode="bilinear").to(x.dtype)
    return F.conv2d(x, sd[p + "conv.weight"], sd[p + "conv.bias"], padding=1)


def sam_mlp3(sd, p, x):
    x = F.relu(_lin(sd, p + "layers.0", x))
    x = F.relu(_lin(sd, p + "layers.1", x))
    return _lin(sd, p + "layers.2", x)


def sam_low_res_masks(sd, cfg, feature_map_i, seg_queries):
    """prompt_encoder(text_embeds=...) + visual_projection + mask_decoder
    (VSM.py:515-533).  feature_map_i [g,g,C]; seg_queries [n,256] -> [n,1,4g,4g]."""
    g = cfg.owl_grid
    n = seg_queries.shape[0]
    sparse = seg_queries.unsqueeze(1)                                        # [n,1,256]
    dense = sd["model.prompt_encoder.no_mask_embed.weight"].reshape(1, -1, 1, 1).expand(n, -1, g, g)
    img = F.linear(feature_map_i.unsqueeze(0), sd["model.visual_projection.weight"]).permute(0, 3, 1, 2)
    pe = dense_pe(sd, g)
    out_tok = torch.cat([sd["model.mask_decoder.iou_token.weight"], sd["model.mask_decoder.mask_tokens.weight"]], 0)
    tokens = torch.cat([out_tok.unsqueeze(0).expand(n, -1, -1), sparse.to(out_tok.dtype)], dim=1)   # [n,6,256]
    src = torch.repeat_interleave(img, n, dim=0) + dense
    pos = torch.repeat_interleave(pe, n, dim=0)
    b, c, h, w = src.shape
    hs, src2 = two_way_transformer(sd, cfg, src, pos, tokens)
    mask_tokens_out = hs[:, 1:5, :]
    src2 = src2.transpose(1, 2).view(b, c, h, w)
    up = sam_upsample(sd, "model.mask_decoder.output_upscaling.0.", src2)
    up = layernorm2d(up, sd["model.mask_decoder.output_upscaling.1.weight"], sd["model.mask_decoder.output_upscaling.1.bias"])
    up = F.gelu(up)
    up = sam_upsample(sd, "model.mask_decoder.output_upscaling.3.", up)
    up = F.gelu(up)
    hyper = torch.stack([sam_mlp3(sd, f"model.mask_decoder.output_hypernetworks_mlps.{i}.", mask_tokens_out[:, i, :]) for i in range(4)], dim=1)
    b, c, h, w = up.shape
    masks = (hyper @ up.view(b, c, h * w)).view(b, 4, h, w)
    return masks[:, 0:1]                                                     # multimask_output=False


# --------------------------------------------------------------------------
# OWL-ViT class / box heads (owlvit.py:63-100,:150-170;
# transformers/models/owlvit/modeling_owlvit.py:1009-1073)
# --------------------------------------------------------------------------
def owl_box_bias(g):
    coords = np.stack(np.meshgrid(np.arange(1, g + 1), np.arange(1, g + 1)), axis=-1).astype(np.float32)
    coords /= np.array([g, g], np.float32)
    coords = torch.from_numpy(coords.reshape(g * g, 2))
    coords = torch.clip(coords, 0.0, 1.0)
    cb = torch.log(coords + 1e-4) - torch.log1p(-coords + 1e-4)
    size = torch.full_like(cb, 1.0 / g)
    sb = torch.log(size + 1e-4) - torch.log1p(-size + 1e-4)
    return torch.cat([cb, sb], dim=-1)                                        # fp32 [g*g,4]


def owl_heads(sd, cfg, feature_map_i, det_queries):
    """OwlViT.forward for n queries on one image: -> (pred_logits [n,g*g,1], pred_boxes [n,g*g,4])."""
    g = cfg.owl_grid
    n = det_queries.shape[0]
    feats = feature_map_i.reshape(1, g * g, -1).repeat(n, 1, 1)
    p = "model.owlvit.class_head."
    ice = _lin(sd, p + "dense0", feats)
    ice = ice / (torch.linalg.norm(ice, dim=-1, keepdim=True) + 1e-6)
    q = det_queries.reshape(n, 1, -1)
    q = q / (torch.linalg.norm(q, dim=-1, keepdim=True) + 1e-6)
    logits = torch.einsum("...pd,...qd->...pq", ice, q)
    shift = _lin(sd, p + "logit_shift", feats)
    scale = F.elu(_lin(sd, p + "logit_scale", feats)) + 1
    logits = (logits + shift) * scale
    p = "model.owlvit.box_head."
    b = _lin(sd, p + "dense2", F.gelu(_lin(sd, p + "dense1", F.gelu(_lin(sd, p + "dense0", feats)))))
    b = b + owl_box_bias(g).to(b.device)   # in-place += in the reference: result stays in activation dtype
    b = b.to(feats.dtype) if feats.dtype != torch.float32 else b
    return logits, torch.sigmoid(b)


# --------------------------------------------------------------------------
# whole-model entry points
# --------------------------------------------------------------------------
def vsm_heads(sd, cfg, hidden, loc_mask, images, original_size, mode="detection"):
    """Everything after the LLM (VSM.py:475-553 / :282-364) for batch 1."""
    seg_all = text_fcs(sd, "seg", hidden)
    det_all = text_fcs(sd, "det", hidden)
    seg_q = seg_all[loc_mask]
    det_q = det_all[loc_mask]
    fmap = owl_visual_embs(sd, cfg, images)
    out = {"seg_queries": seg_q, "det_queries": det_q, "feature_map": fmap}
    low = sam_low_res_masks(sd, cfg, fmap[0], seg_q)
    out["low_res_masks"] = low
    pm = F.interpolate(low.float(), tuple(original_size), mode="bilinear", align_corners=False)
    out["pred_masks"] = pm[:, 0]
    if mode == "segmentation":
        return out
    logits, boxes = owl_heads(sd, cfg, fmap[0], det_q)
    out["pred_logits"], out["pred_boxes"] = logits, boxes
    return out


def model_forward_inference(sd, cfg, images, images_clip, input_ids, original_size):
    """VSMForCausalLM.model_forward(inference=True) (VSM.py:201-364): teacher-forced
    single pass; `input_ids` already contains the answer with [LOC]."""
    m = input_ids[:, 1:] == cfg.loc_token_idx
    m = torch.cat([m, torch.zeros((m.shape[0], 1), dtype=torch.bool, device=m.device)], dim=1)
    loc_mask = torch.cat([torch.zeros((m.shape[0], 255), dtype=torch.bool, device=m.device), m], dim=1)
    logits, hidden = lm_forward(sd, cfg, input_ids, images_clip)
    out = vsm_heads(sd, cfg, hidden, loc_mask, images, original_size)
    out["hidden"], out["logits"] = hidden, logits
    return out


def vsm_inference(sd, cfg, images_clip, images, input_ids, original_size, max_new_tokens=100,
                  mode="detection", eos_token_id=2, forced_ids=None):
    """VSMForCausalLM.inference (VSM.py:438-553) with the restated greedy loop."""
    out_ids, hidden, argmaxes = greedy_generate(sd, cfg, input_ids, images_clip, max_new_tokens, eos_token_id, forced_ids)
    if mode == "vqa":
        return {"output_ids": out_ids, "argmaxes": argmaxes}
    loc_mask = loc_mask_from_output_ids(out_ids, cfg.loc_token_idx)
    out = vsm_heads(sd, cfg, hidden, loc_mask, images, original_size, mode)
    out["output_ids"], out["argmaxes"], out["hidden"] = out_ids, argmaxes, hidden
    return out


# --------------------------------------------------------------------------
# host-side image preprocessing
#   /root/reference/visual_search.py:186-194; VisualSearch/utils/utils.py:28-39;
#   transformers CLIPImageProcessor defaults (shortest edge 224 bicubic, center
#   crop 224, /255, CLIP mean/std) and OwlViTImageProcessor defaults (resize to
#   768x768 bicubic, /255, CLIP mean/std;
#   transformers/models/owlvit/image_processing_owlvit.py:103-113)
# --------------------------------------------------------------------------
CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def expand2square(pil_img, background_color):
    from PIL import Image
    width, height = pil_img.size
    if width == height:
        return pil_img
    side = max(width, height)
    result = Image.new(pil_img.mode, (side, side), background_color)
    result.paste(pil_img, (0, 0))
    return result


def _normalize(arr_u8):
    x = arr_u8.astype(np.float32) * np.float32(1 / 255.0)
    x = (x - np.array(CLIP_MEAN, np.float32)) / np.array(CLIP_STD, np.float32)
    return torch.from_numpy(np.ascontiguousarray(x.transpose(2, 0, 1)))


def preprocess_clip(pil_img, size=224):
    from PIL import Image
    bg = tuple(int(x * 255) for x in CLIP_MEAN)
    img = expand2square(pil_img.convert("RGB"), bg)
    w, h = img.size
    short = min(w, h)
    nw, nh = int(w * size / short), int(h * size / short)
    img = img.resize((nw, nh), resample=Image.BICUBIC)
    left, top = (nw - size) // 2, (nh - size) // 2
    img = img.crop((left, top, left + size, top + size))
    return _normalize(np.array(img)).unsqueeze(0)


def preprocess_owl(pil_img, size=768):
    from PIL import Image
    img = pil_img.convert("RGB").resize((size, size), resample=Image.BICUBIC)
    return _normalize(np.array(img)).unsqueeze(0)


# --------------------------------------------------------------------------
# search controller (restated from /root/reference/visual_search.py:227-283,
# :378-516).  `vsm` is any object with .inference(image, question, mode).
# --------------------------------------------------------------------------
def split_4subpatches(bbox):
    r = bbox[3] / bbox[2]
    if r >= 2:
        return 1, 4
    elif r <= 0.5:
        return 4, 1
    return 2, 2


def get_sub_patches(bbox, nw, nh):
    ws = int(bbox[2] // nw)
    hs = int(bbox[3] / nh)
    out = []
    for j in range(nh):
        for i in range(nw):
            sw = bbox[2] - i * ws if i == nw - 1 else ws
            sh = bbox[3] - j * hs if j == nh - 1 else hs
            out.append([bbox[0] + i * ws, bbox[1] + j * hs, sw, sh])
    return out, ws, hs


def get_subpatch_scores(hm, bbox, subs):
    total = (hm / (bbox[2] * bbox[3])).sum()
    scores = []
    for sp in subs:
        b = [sp[0] - bbox[0], sp[1] - bbox[1], sp[2], sp[3]]
        s = (hm[b[1]:b[1] + b[3], b[0]:b[0] + b[2]] / (bbox[2] * bbox[3])).sum()
        if total > 0:
            s /= total
        else:
            s *= 0
        scores.append(s)
    return scores


def normalize_score(hm):
    mx, mn = hm.max(), hm.min()
    if mx != mn:
        return (hm - mn) / (mx - mn)
    return hm * 0


@functools.total_ordering
class Prioritize:
    def __init__(self, priority, item):
        self.priority, self.item = priority, item

    def __eq__(self, other):
        return self.priority == other.priority

    def __lt__(self, other):
        return self.priority < other.priority


def visual_search(vsm, image, target_object_name, target_bbox, smallest_size, confidence_high=0.5,
                  confidence_low=0.3, target_cue_threshold=6.0, target_cue_threshold_decay=0.7,
                  target_cue_threshold_minimum=3.0, extract_noun_chunks=None):
    """Recursion-for-recursion restatement of visual_search / visual_search_queue."""
    import copy
    init = {"bbox": [0, 0, image.width, image.height], "scale_level": 1, "score": None, "parent_index": -1}
    search_path = [init]
    queue = PriorityQueue()

    def rec(cur):
        bb = cur["bbox"]
        lvl = cur["scale_level"]
        patch = image.crop((int(bb[0]), int(bb[1]), int(bb[0] + bb[2]), int(bb[1] + bb[3])))
        q = "Please locate the {} in this image.".format(target_object_name)
        boxes, logits, hm = vsm.inference(copy.deepcopy(patch), q, mode="detection")
        if len(logits) > 0:
            ti = logits.view(-1).argmax()
            tl = logits.view(-1).max()
            fb = boxes[ti].view(4)
            fb = fb * torch.Tensor([patch.width, patch.height, patch.width, patch.height])
            fb[:2] -= fb[2:] / 2
            if tl > confidence_high:
                search_path[-1]["detection_result"] = fb
                if len(search_path) == 1:
                    av = boxes[logits.view(-1) > 0.5].view(-1, 4)
                    av = av * torch.Tensor([[patch.width, patch.height, patch.width, patch.height]])
                    av[:, :2] -= av[:, 2:] / 2
                    return True, av
                return True, None
            else:
                search_path[-1]["temp_detection_result"] = (tl, fb)
        if min(bb[2], bb[3]) <= smallest_size:
            return False, None
        hm = hm.view(bb[3], bb[2], 1)
        score_max = hm.max().item()
        thr = max(target_cue_threshold_minimum, target_cue_threshold * target_cue_threshold_decay ** (lvl - 1))
        if score_max > thr:
            final = normalize_score(hm)
        else:
            q = ("According to the common sense knowledge and possible visual cues, what is the most likely "
                 "location of the {} in the image?").format(target_object_name)
            vqa = vsm.inference(copy.deepcopy(patch), q, mode="vqa")
            phrase = vqa.split("most likely to appear")[-1].strip()
            if phrase.endswith("."):
                phrase = phrase[:-1]
            phrase = phrase.split(target_object_name)[-1]
            chunks = extract_noun_chunks(phrase) if extract_noun_chunks else []
            phrase = chunks[0] if len(chunks) == 1 else "region {}".format(phrase)
            q = "Please locate the {} in this image.".format(phrase)
            final = normalize_score(vsm.inference(copy.deepcopy(patch), q, mode="segmentation").view(bb[3], bb[2], 1))
        idx = len(search_path) - 1
        if score_max <= thr:
            search_path[idx]["context_cue"] = vqa + "#" + phrase
        search_path[idx]["final_heatmap"] = final.cpu().numpy()
        subs, _, _ = get_sub_patches(bb, *split_4subpatches(bb))
        tmp = cur
        sc = [0] * len(subs)
        while True:
            ts = get_subpatch_scores(tmp["final_heatmap"], tmp["bbox"], subs)
            sc = [sc[i] + ts[i] / (4 ** tmp["scale_level"]) for i in range(len(sc))]
            if tmp["parent_index"] == -1:
                break
            tmp = search_path[tmp["parent_index"]]
        for sp, s in zip(subs, sc):
            queue.put(Prioritize(-s, {"bbox": sp, "scale_level": lvl + 1, "score": s, "parent_index": idx}))
        while not queue.empty():
            nxt = queue.get().item
            search_path.append(nxt)
            ok, av = rec(nxt)
            if ok:
                return ok, av
        return False, None

    ok, all_valid = rec(init)
    path_length = len(search_path)
    final_step = search_path[-1]
    if not ok:
        max_logit, final_step, path_length = 0, None, 0
        for i, st in enumerate(search_path):
            if "temp_detection_result" in st and st["temp_detection_result"][0] > max_logit:
                max_logit, final_step, path_length = st["temp_detection_result"][0], st, i + 1
        final_step["detection_result"] = final_step["temp_detection_result"][1]
        if max_logit >= confidence_low:
            ok = True
    return final_step, path_length, ok, all_valid, search_path


