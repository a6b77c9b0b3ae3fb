"""VSM engine: the per-crop model evaluation of the V* guided visual search, batched over the crop
frontier, executed entirely by the hand-written sm_90a kernels behind include/vstar_b200.h.

Mirrors /root/reference/VisualSearch/model/VSM.py `VSMForCausalLM.inference` / `.model_forward(inference=True)`
(:438-553, :201-364) with the restructurings SURVEY.md §2b calls out:
  * frontier batching: B crops share every GEMM (M = B*T) instead of batch 1;
  * the answer is DRAFT-VERIFIED in one prefill (teacher-force the draft "Sure, [LOC] ." and check the greedy
    argmax at every answer position) instead of `generate(use_cache=False)` re-running CLIP + the whole 7B
    for each of the ~6 tokens (VSM.py:451-458); a mismatch falls back to exact step-by-step greedy decoding
    on the fused-QKV cache, so the emitted ids are always the reference's greedy ids;
  * lm_head / text_hidden_fcs run only on the rows that are consumed (VSM.py:475-490 run them on all T rows);
  * CLIP stops at the layer that `select_layer=-2` reads (clip_encoder.py:31-39);
  * dense positional encoding, box bias and the prompt tokens are constants built once at load.

torch is used for device memory, streams and a few index/slice views only.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass

import numpy as np
import torch

from . import ops
from .config import VSMConfig, IMAGE_TOKEN_INDEX

BF = torch.bfloat16


def _pad8(n):
    return (n + 7) // 8 * 8


class CoreWeights:
    """Llama-7B + CLIP ViT-L/14 + mm_projector: shared by the VSM (visual search model) and the SEAL VQA LLM.
    Device-resident weights re-laid-out for the kernels (fused QKV, interleaved gate/up).  Source = any callable
    name -> CPU/GPU tensor in the reference's state_dict key layout (SURVEY.md §8f-3).
    dtype: torch.bfloat16 (default; the VSM) or torch.float16 (the SEAL VQA LLM as the reference runs it); the engine built on
    these weights computes in that dtype."""

    def __init__(self, cfg: VSMConfig, get, device="cuda", dtype=BF, quant=None):
        if dtype not in (torch.bfloat16, torch.float16):
            raise ValueError(f"weights dtype must be torch.bfloat16 or torch.float16, got {dtype}")
        if quant not in (None, "nf4") or (quant == "nf4" and dtype != torch.float16):
            raise ValueError(f"quant must be None or 'nf4' (fp16 weights only), got {quant!r} with {dtype}")
        self.cfg = cfg
        self.device = device
        self.dtype = dtype
        self.quant = quant
        dev = device

        def g(name):
            return get(name).to(device=dev, dtype=dtype).contiguous()

        def lin(name):
            """a Linear weight: NF4 when quantised, straight from the fp16 copy so that only one fp16 tensor is resident"""
            return ops.nf4_quantize(g(name)) if quant else g(name)

        self._g = g
        self._lin = lin
        c = cfg
        # ---- Llama
        self.embed = g("model.embed_tokens.weight")
        self.lm_head = g("lm_head.weight")
        self.final_norm = g("model.norm.weight")
        self.layers = []
        # NF4 quantises each HF tensor on its own, so the norms cannot be folded into the weights first
        self.fold_norms = os.environ.get("VSB_FOLD_NORMS", "1") != "0" and not quant
        ones = None
        for i in range(c.n_layers):
            p = f"model.layers.{i}."
            if quant:
                self.layers.append(dict(
                    wqkv=ops.NF4Weight.cat_rows([lin(p + "self_attn.q_proj.weight"), lin(p + "self_attn.k_proj.weight"),
                                                 lin(p + "self_attn.v_proj.weight")]),
                    wo=lin(p + "self_attn.o_proj.weight"),
                    wgu=ops.NF4Weight.interleave_rows(lin(p + "mlp.gate_proj.weight"), lin(p + "mlp.up_proj.weight")),
                    wdown=lin(p + "mlp.down_proj.weight"),
                    ln1=g(p + "input_layernorm.weight"), ln2=g(p + "post_attention_layernorm.weight")))
                continue
            wqkv = torch.cat([g(p + "self_attn.q_proj.weight"), g(p + "self_attn.k_proj.weight"), g(p + "self_attn.v_proj.weight")], 0)
            gate, up = g(p + "mlp.gate_proj.weight"), g(p + "mlp.up_proj.weight")
            wgu = torch.stack([gate, up], dim=1).reshape(2 * c.intermediate, c.hidden).contiguous()   # row 2j = gate_j, 2j+1 = up_j
            del gate, up
            ln1, ln2 = g(p + "input_layernorm.weight"), g(p + "post_attention_layernorm.weight")
            if self.fold_norms:
                # LlamaRMSNorm's weight folded into the consuming projections: w * (x * rstd) @ W^T == rstd * (x @ (W * w)^T).  The
                # kernels then apply 1/rms in the GEMM epilogue (vsb_gemm_rowscale_bf16) and no norm kernel runs; ln1 / ln2 become
                # ones so that the unfused decode path (skinny GEMMs) computes the same function from the same folded weights.
                wqkv = (wqkv.float() * ln1.float()[None, :]).to(dtype)
                wgu = (wgu.float() * ln2.float()[None, :]).to(dtype)
                if ones is None:
                    ones = torch.ones_like(ln1)
                ln1 = ln2 = ones
            self.layers.append(dict(wqkv=wqkv.contiguous(), wo=g(p + "self_attn.o_proj.weight"), wgu=wgu.contiguous(),
                                    wdown=g(p + "mlp.down_proj.weight"), ln1=ln1, ln2=ln2))
        # RoPE tables exactly as HF builds them (fp32 outer product -> cos/sin -> the model dtype)
        hd = c.head_dim
        inv = 1.0 / (c.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.float32) / hd))
        fr = torch.outer(torch.arange(2048, dtype=torch.float32), inv)
        self.rope_cos = fr.cos().to(dtype).to(dev).contiguous()
        self.rope_sin = fr.sin().to(dtype).to(dev).contiguous()
        # ---- ViTs
        self.clip = self._vit(g, "model.vision_tower.vision_tower.vision_model.", c.clip_layers + 1 + c.clip_select_layer
                              if c.clip_select_layer < 0 else c.clip_select_layer, c.clip_patch, "pre_layrnorm")
        self.mm_w, self.mm_b = lin("model.mm_projector.weight"), g("model.mm_projector.bias")

    @classmethod
    def from_state_dict(cls, cfg, sd, device="cuda", dtype=BF, **kw):
        return cls(cfg, lambda n: sd[n], device, dtype=dtype, **kw)

    def linear_bytes(self):
        """device bytes of the Llama and projector Linear weights (the ones NF4 quantises)"""
        nb = ops.weight_nbytes
        return sum(nb(L[k]) for L in self.layers for k in ops.NF4_LINEARS) + nb(self.mm_w)

    @staticmethod
    def _vit(g, p, n_layers, patch, pre_name):
        pw = g(p + "embeddings.patch_embedding.weight")
        C = pw.shape[0]
        K = 3 * patch * patch
        Kp = _pad8(K)
        w = torch.zeros((C, Kp), dtype=pw.dtype, device=pw.device)
        w[:, :K] = pw.reshape(C, K)
        layers = []
        for i in range(n_layers):
            q = f"{p}encoder.layers.{i}."
            layers.append(dict(
                wqkv=torch.cat([g(q + "self_attn.q_proj.weight"), g(q + "self_attn.k_proj.weight"), g(q + "self_attn.v_proj.weight")], 0).contiguous(),
                bqkv=torch.cat([g(q + "self_attn.q_proj.bias"), g(q + "self_attn.k_proj.bias"), g(q + "self_attn.v_proj.bias")], 0).contiguous(),
                wo=g(q + "self_attn.out_proj.weight"), bo=g(q + "self_attn.out_proj.bias"),
                ln1=(g(q + "layer_norm1.weight"), g(q + "layer_norm1.bias")), ln2=(g(q + "layer_norm2.weight"), g(q + "layer_norm2.bias")),
                w1=g(q + "mlp.fc1.weight"), b1=g(q + "mlp.fc1.bias"), w2=g(q + "mlp.fc2.weight"), b2=g(q + "mlp.fc2.bias")))
        return dict(patch_w=w, Kpad=Kp, cls=g(p + "embeddings.class_embedding"), pos=g(p + "embeddings.position_embedding.weight"),
                    pre=(g(p + pre_name + ".weight"), g(p + pre_name + ".bias")), layers=layers, C=C)


class VSMWeights(CoreWeights):
    """+ OWL-ViT-B/16, OWL heads, [LOC] query MLPs, SAM prompt encoder / mask decoder (stacked class-head rows,
    permuted conv taps)."""

    def __init__(self, cfg: VSMConfig, get, device="cuda", dtype=BF, quant=None):
        if dtype != BF:
            raise ValueError("the VSM runs in bf16 only, as in the reference (visual_search.py:145)")
        if quant is not None:
            raise ValueError("the VSM is not quantised: the reference loads it in bf16 only")
        super().__init__(cfg, get, device)
        g, c, dev = self._g, cfg, device
        self.owl = self._vit(g, "model.owlvit.vision_model.", c.owl_layers, c.owl_patch, "pre_layernorm")
        self.owl["post_w"], self.owl["post_b"] = g("model.owlvit.vision_model.post_layernorm.weight"), g("model.owlvit.vision_model.post_layernorm.bias")
        self.owl["merge_w"], self.owl["merge_b"] = g("model.owlvit.layer_norm.weight"), g("model.owlvit.layer_norm.bias")
        # ---- OWL heads: class head rows stacked [dense0 ; logit_shift ; logit_scale]
        ch = "model.owlvit.class_head."
        self.cls_w = torch.cat([g(ch + "dense0.weight"), g(ch + "logit_shift.weight"), g(ch + "logit_scale.weight")], 0).contiguous()
        self.cls_b = torch.cat([g(ch + "dense0.bias"), g(ch + "logit_shift.bias"), g(ch + "logit_scale.bias")], 0).contiguous()
        bh = "model.owlvit.box_head."
        self.box = [(g(bh + f"dense{i}.weight"), g(bh + f"dense{i}.bias")) for i in range(3)]
        self.box_bias = self._box_bias(c.owl_grid).to(dev)
        # ---- query MLPs
        self.fcs = {}
        for w in ("seg", "det"):
            p = f"model.text_hidden_fcs_{w}.0."
            self.fcs[w] = (g(p + "0.weight"), g(p + "0.bias"), g(p + "2.weight"), g(p + "2.bias"))
        # ---- SAM prompt encoder / mask decoder
        self.vp_w = g("model.visual_projection.weight")
        self.no_mask = g("model.prompt_encoder.no_mask_embed.weight").view(-1).contiguous()
        self.dense_pe = self._dense_pe(g("model.prompt_encoder.pe_layer.positional_encoding_gaussian_matrix"), c.owl_grid)
        md = "model.mask_decoder."
        self.out_tokens = torch.cat([g(md + "iou_token.weight"), g(md + "mask_tokens.weight")], 0).contiguous()   # [5,256]
        t = md + "transformer."

        def att(p):
            return dict(wq=g(p + "q_proj.weight"), bq=g(p + "q_proj.bias"), wk=g(p + "k_proj.weight"), bk=g(p + "k_proj.bias"),
                        wv=g(p + "v_proj.weight"), bv=g(p + "v_proj.bias"), wo=g(p + "out_proj.weight"), bo=g(p + "out_proj.bias"))

        self.sam_layers = []
        for i in range(c.sam_depth):
            lp = f"{t}layers.{i}."
            L = dict(self_attn=att(lp + "self_attn."), t2i=att(lp + "cross_attn_token_to_image."), i2t=att(lp + "cross_attn_image_to_token."),
                     w1=g(lp + "mlp.lin1.weight"), b1=g(lp + "mlp.lin1.bias"), w2=g(lp + "mlp.lin2.weight"), b2=g(lp + "mlp.lin2.bias"))
            for n in ("norm1", "norm2", "norm3", "norm4"):
                L[n] = (g(lp + n + ".weight"), g(lp + n + ".bias"))
            self.sam_layers.append(L)
        self.sam_final = att(t + "final_attn_token_to_image.")
        self.sam_final_norm = (g(t + "norm_final_attn.weight"), g(t + "norm_final_attn.bias"))
        # 3x3 convs: [Cout, Cin, 3, 3] -> [Cout, ky, kx, Cin] to match the NHWC im2col
        self.up0_w = g(md + "output_upscaling.0.conv.weight").permute(0, 2, 3, 1).reshape(c.sam_dim // 4, -1).contiguous()
        self.up0_b = g(md + "output_upscaling.0.conv.bias")
        self.up_ln = (g(md + "output_upscaling.1.weight"), g(md + "output_upscaling.1.bias"))
        self.up1_w = g(md + "output_upscaling.3.conv.weight").permute(0, 2, 3, 1).reshape(c.sam_dim // 8, -1).contiguous()
        self.up1_b = g(md + "output_upscaling.3.conv.bias")
        hp = md + "output_hypernetworks_mlps.0.layers."     # mask token 0 only (multimask_output=False)
        self.hyper = [(g(hp + f"{j}.weight"), g(hp + f"{j}.bias")) for j in range(3)]

    @staticmethod
    def _box_bias(gsz):
        # /root/reference/VisualSearch/model/owlvit/owlvit.py:42-77 (fp32 numpy/torch constant)
        coords = np.stack(np.meshgrid(np.arange(1, gsz + 1), np.arange(1, gsz + 1)), axis=-1).astype(np.float32)
        coords /= np.array([gsz, gsz], np.float32)
        coords = torch.clip(torch.from_numpy(coords.reshape(gsz * gsz, 2)), 0.0, 1.0)
        cb = torch.log(coords + 1e-4) - torch.log1p(-coords + 1e-4)
        size = torch.full_like(cb, 1.0 / gsz)
        sb = torch.log(size + 1e-4) - torch.log1p(-size + 1e-4)
        return torch.cat([cb, sb], dim=-1).contiguous()

    @staticmethod
    def _dense_pe(G, gsz):
        """PositionEmbeddingRandom.forward (prompt_encoder.py:203-229) evaluated ONCE, with the same torch ops in
        the buffer's dtype (bf16 after from_pretrained(torch_dtype=bf16)) so the constant is bit-identical."""
        grid = torch.ones((gsz, gsz), device=G.device, dtype=G.dtype)
        y = (grid.cumsum(dim=0) - 0.5) / gsz
        x = (grid.cumsum(dim=1) - 0.5) / gsz
        cxy = torch.stack([x, y], dim=-1)
        cxy = 2 * cxy - 1
        cxy = cxy @ G
        cxy = 2 * np.pi * cxy
        pe = torch.cat([torch.sin(cxy), torch.cos(cxy)], dim=-1)      # [g,g,256]
        return pe.reshape(gsz * gsz, -1).contiguous()



@dataclass
class CropResult:
    """Per-crop outputs of one detection-mode evaluation (device tensors)."""
    output_ids: list
    low_res: torch.Tensor        # [n_loc, 4g, 4g] fp32
    logits: torch.Tensor         # [n_loc, g*g] fp32 (pre-sigmoid)
    scores: torch.Tensor         # [n_loc, g*g] fp32 (sigmoid)
    boxes: torch.Tensor          # [n_loc, g*g, 4] fp32 cxcywh
    verified: bool


class LlamaClipCore:
    """CLIP tower + Llama decoder on the sm_90a kernels with the fused-QKV cache; base of VSMEngine and VQAEngine.
    Computes in the weights' dtype (bf16, or fp16 for the VQA engine): cache, scratch and activations follow it."""

    MAX_POSITIONS = 2048          # rows of the RoPE tables (Llama-1 / Vicuna max_position_embeddings)

    def __init__(self, weights: CoreWeights, max_batch=8, max_tokens=384):
        self.w = weights
        self.cfg = weights.cfg
        self.dev = weights.device
        self.dtype = weights.dtype
        # rows per KV-cache slot allocated up front; the cache GROWS (up to MAX_POSITIONS) when a prompt or a generation
        # needs more - nothing is truncated silently, and a sequence beyond the RoPE tables raises VsbError
        self.max_tokens = min(int(max_tokens), self.MAX_POSITIONS)
        self._cache = None
        self._cache_shape = None
        self._layer_table = None        # ctypes array of per-layer weight pointers for the native layer runner
        self.stats = dict(verified=0, fallback=0, prefix_shared=0)
        # shared-prefix KV (see prefill): the text before <im_start> is the same for every crop
        self.prefix_cache = True
        self.tail_only = os.environ.get("VSB_TAIL_ONLY", "1") != "0"    # last layer over the consumed rows only (draft-verify path)
        # detection logits / scores / boxes rounded to bf16 VALUES like the reference's bf16 model emits them, so thresholds,
        # argmax ties and all_valid_boxes are decided on the same numbers (visual_search.py:399-409); False = full fp32 heads
        self.heads_bf16 = True
        self._prefix_ids = None          # tuple of token ids
        self._prefix_kv = None           # [n_layers, P, 3d] snapshot of the cache rows of that prefix
        self._prefix_slots = 0           # cache slots whose rows 0..P currently hold it
        self._P = 0                      # prefix rows omitted from the residual stream returned by the last prefill
        self._Tn = 0
        self._consts = {}                # small index tensors on the device, built once per shape (also keeps graph capture clean)
        # CUDA graphs for small frontier batches (VSMEngine.inference): a single crop is ~1400 kernels of a few microseconds,
        # i.e. bound by the host's launch rate, not by the GPU; replaying one captured graph removes that (DESIGN.md)
        self.graph_max_batch = int(os.environ.get("VSB_GRAPH_MAX_BATCH", "8"))
        self._graphs = {}
        self._graph_seen = {}
        self._capturing = False

    def _const(self, key, values, dtype=torch.int64):
        """device tensor of a small host list, cached by key (pure function of the call's shape parameters)"""
        t = self._consts.get(key)
        if t is None:
            if self._capturing:
                raise RuntimeError(f"device constant {key!r} requested for the first time during graph capture")
            if len(self._consts) > 512:
                self._consts.clear()
            t = torch.tensor(values, dtype=dtype).to(self.dev)
            self._consts[key] = t
        return t

    # ------------------------------------------------------------------ ViT
    def _vit_forward(self, vw, pixels, patch, heads, image, eps):
        """pixels [B,3,S,S] bf16 -> residual stream after the last executed layer [B*Ntok, C]"""
        c = self.cfg
        B = pixels.shape[0]
        g = image // patch
        S = g * g + 1
        C = vw["C"]
        A = ops.patchify(pixels, patch, vw["Kpad"])
        x = torch.empty((B * S, C), dtype=self.dtype, device=self.dev)
        ops.gemm(A, vw["patch_w"], out=x, rows_per_group=g * g, group_stride=S, group_offset=1)
        ops.vit_add_pos_(x, vw["cls"], vw["pos"], B, S)
        x = ops.layernorm(x, vw["pre"][0], vw["pre"][1], eps)
        hd = C // heads
        for L in vw["layers"]:
            h = ops.layernorm(x, L["ln1"][0], L["ln1"][1], eps)
            qkv = ops.gemm(h, L["wqkv"], bias=L["bqkv"])
            a = ops.attn_fused_qkv(qkv, B, S, heads, hd, False, hd ** -0.5)
            x = ops.gemm(a, L["wo"], bias=L["bo"], residual=x)
            h = ops.layernorm(x, L["ln2"][0], L["ln2"][1], eps)
            h = ops.gemm(h, L["w1"], bias=L["b1"], epilogue=ops.EPI_QUICK_GELU)
            x = ops.gemm(h, L["w2"], bias=L["b2"], residual=x)
        return x, S

    def clip_tokens(self, images_clip):
        """-> hidden_states[select_layer] incl. CLS: [B*257, C] (feature_select drops CLS afterwards)"""
        c = self.cfg
        return self._vit_forward(self.w.clip, images_clip, c.clip_patch, c.clip_heads, c.clip_image, c.vit_eps)

    def owl_feature_map(self, images):
        """OwlViT.get_visual_embs -> [B*g*g, C]"""
        c = self.cfg
        x, S = self._vit_forward(self.w.owl, images, c.owl_patch, c.owl_heads, c.owl_image, c.vit_eps)
        o = self.w.owl
        return ops.owl_merge(x, o["post_w"], o["post_b"], o["merge_w"], o["merge_b"], images.shape[0], S, c.vit_eps)

    # ------------------------------------------------------------------ LLM
    def _capacity(self, need):
        """rows per cache slot for a sequence of `need` positions: at least self.max_tokens, multiples of 64"""
        if need > self.MAX_POSITIONS:
            raise ops._lib.VsbError(f"sequence of {need} positions exceeds the {self.MAX_POSITIONS} rows of the RoPE tables "
                                    "(max_position_embeddings of the Llama-1/Vicuna backbone)")
        return min(self.MAX_POSITIONS, max(self.max_tokens, (need + 63) // 64 * 64))

    def _ensure_cache(self, B, Tmax, keep=False):
        """cache with >= B slots of >= Tmax rows.  keep=True preserves the rows already written (decode-time growth)."""
        c = self.cfg
        cur = self._cache_shape
        if self._cache is not None and cur[1] >= B and cur[2] >= Tmax:
            return self._cache
        if cur is not None:
            B, Tmax = max(B, cur[1]), max(Tmax, cur[2])
        shape = (c.n_layers, B, Tmax, 3 * c.hidden)
        old = self._cache if keep else None
        self._cache = None                                # release before allocating the replacement (unless kept)
        self._cache = torch.empty(shape, dtype=self.dtype, device=self.dev)
        if old is not None:
            self._cache[:, :cur[1], :cur[2]].copy_(old)
        self._cache_shape = shape
        self._prefix_slots = 0
        self._graphs.clear()            # captured graphs hold pointers into the old cache
        self._graph_seen.clear()
        return self._cache

    def _llm_layers(self, x, B, Tn, past, positions=None, k_start=None, cache_row_offset=0, tail_rows=0, q_seg=None, seg_lo=0):
        """Run all decoder layers over the Tn new rows per sequence in x [B*Tn, d] (in place on the residual stream).
        Fused q|k|v rows live in the per-layer cache [B, Tmax, 3d] at positions past..past+Tn.  One native call
        (csrc/llama_layers.cu) sequences the 8 kernels of every layer: RMSNorm, QKV GEMM writing cache rows, RoPE in
        place, attention through strides, o-proj + residual, RMSNorm, gate|up GEMM with SwiGLU epilogue, down + residual."""
        c = self.cfg
        if self._layer_table is None:
            self._layer_table = ops.llama_layer_table(self.w.layers)
        Bc, Tm = self._cache_shape[1], self._cache_shape[2]
        scratch = torch.empty((B * Tn * (2 * c.hidden + c.intermediate),), dtype=self.dtype, device=self.dev)
        deq = None
        if getattr(self.w, "quant", None):
            # NF4 projections dequantise into this buffer on the row counts that take the tile kernels
            deq = torch.empty((2 * c.intermediate * c.hidden,), dtype=self.dtype, device=self.dev)
        return ops.llama_layers(self._layer_table, len(self.w.layers), x, B, Tn, past, self._cache, Bc, Tm, c.hidden, c.n_heads,
                                c.intermediate, c.rms_eps, self.w.rope_cos, self.w.rope_sin, scratch, positions=positions,
                                k_start=k_start, cache_row_offset=cache_row_offset, tail_rows=tail_rows, q_seg=q_seg, seg_lo=seg_lo,
                                norm_folded=getattr(self.w, "fold_norms", False), deq_scratch=deq)

    def _logits_rows(self, x, rows):
        """final RMSNorm + lm_head on selected rows of the residual stream -> (hidden [n,d], argmax [n], logits fp32 [n,V])"""
        c = self.cfg
        sel = ops.gather_rows(rows, x)
        hn = ops.rmsnorm(sel, self.w.final_norm, c.rms_eps)
        logits = ops.gemm(hn, self.w.lm_head, out_dtype=torch.float32)
        idx, _ = ops.argmax_rows(logits)
        return hn, idx, logits

    def x_row(self, b, pos):
        """row of the residual stream returned by the last prefill() that holds spliced position `pos` of crop `b`"""
        assert pos >= self._P, "position inside the shared prefix: its rows are not recomputed"
        return b * self._Tn + pos - self._P

    def prefill(self, input_ids, images_clip, tail_rows=0, reserve=0, ids_dev=None):
        """input_ids int64 [B, L] (same L and same image position for the whole batch), images_clip [B,3,224,224] bf16.
        tail_rows > 0: the caller reads only the last tail_rows positions of every crop (see vsb_llama_layers).
        reserve: positions the caller will append by decoding (the cache slot is sized for T + reserve up front).
        Returns (x, T, img_pos): the residual stream (pre final norm) of the rows that were computed, the spliced length T
        and the image position.  Use x_row(b, pos) to address x.

        Shared prefix: the tokens before <im_start> (the conversation's system prompt and "USER:",
        conversation.py:355-365) are identical for every crop and, the model being causal, so are their K/V rows.  The
        first prefill with a given prefix computes everything and snapshots those cache rows; later calls copy them into
        the batch slots that lack them and run the decoder only over the T - P rows from <im_start> on (past = P).
        Every remaining row sees bit-identical inputs, so the result is the unshared one, ~11 % fewer 7B FLOPs per crop.
        `self.prefix_cache = False` switches it off."""
        c = self.cfg
        B, L = input_ids.shape
        # all id bookkeeping on the host copy: nothing below may wait for the GPU (callers pipeline chunks, VSM._run)
        input_ids = input_ids if input_ids.device.type == "cpu" else input_ids.cpu()
        pos = (input_ids[0] == IMAGE_TOKEN_INDEX).nonzero()
        assert pos.numel() == 1, "exactly one <image> placeholder expected (llava_arch.py:185-208)"
        img_pos = int(pos[0, 0])
        assert bool((input_ids[:, img_pos] == IMAGE_TOKEN_INDEX).all())
        n_img = c.clip_tokens
        T = L - 1 + n_img
        assert img_pos >= 1
        self._ensure_cache(B, self._capacity(T + reserve))
        # P = rows before the <im_start> slot (the CLS row of the projector GEMM lands on that slot, see below)
        P = 0
        if self.prefix_cache and img_pos >= 2:
            head = input_ids[:, :img_pos - 1]
            if bool((head == head[0]).all()):
                pid = tuple(head[0].tolist())
                if pid == self._prefix_ids:
                    P = len(pid)
                else:                                   # new prefix: this call computes it in full and snapshots it below
                    self._prefix_ids, self._prefix_kv, self._prefix_slots = None, None, 0
        Tn = T - P
        ct, S = self.clip_tokens(images_clip)                       # [B*257, Cc]
        x = torch.empty((B * Tn, c.hidden), dtype=self.dtype, device=self.dev)
        # mm_projector over all B*257 rows in ONE GEMM whose epilogue scatters each crop's rows straight into the LLM
        # input buffer: patch row i of crop b -> x[b*Tn + img_pos - P + i].  The CLS row lands on the <im_start> slot
        # (img_pos - 1 >= P) and is overwritten by the embedding splice below.
        ops.gemm(ct, self.w.mm_w, out=x, bias=self.w.mm_b, rows_per_group=S, group_stride=Tn, group_offset=img_pos - 1 - P)
        # ids_dev: the caller already holds input_ids[:, P:] on the device (static buffer of a captured graph)
        ids_new = ids_dev if ids_dev is not None else (input_ids[:, P:] if P else input_ids).contiguous().to(self.dev, non_blocking=True)
        ops.embed_splice(ids_new, self.w.embed, x, img_pos - P, n_img)
        if P:
            if self._prefix_slots < B:                  # slots that do not hold the prefix rows yet
                assert not self._capturing, "prefix rows must be in place before a graph is captured"
                self._cache[:, self._prefix_slots:B, :P].copy_(self._prefix_kv[:, None])
                self._prefix_slots = B
            self.stats["prefix_shared"] += B
        self._llm_layers(x, B, Tn, P, tail_rows=tail_rows if self.tail_only else 0)
        if not P:
            # a full prefill has just overwritten rows 0.. of slots 0..B-1: whatever prefix they held is gone
            self._prefix_slots = 0
            if self.prefix_cache and img_pos >= 2 and self._prefix_ids is None:
                head = input_ids[:, :img_pos - 1]
                if bool((head == head[0]).all()):
                    self._prefix_ids = tuple(head[0].tolist())
                    self._prefix_kv = self._cache[:, 0, :img_pos - 1].clone()
                    self._prefix_slots = B              # every slot of this batch just computed the same rows
        self._P, self._Tn = P, Tn
        return x, T, img_pos

    def decode_step(self, tokens, B, past):
        """one greedy step for B sequences that all have `past` cached positions; tokens int64 [B] -> next argmax [B]"""
        c = self.cfg
        if past + 1 > self._cache_shape[2]:
            self._ensure_cache(self._cache_shape[1], self._capacity(past + 64), keep=True)
        x = ops.gather_rows(tokens.contiguous(), self.w.embed)
        self._llm_layers(x, B, 1, past)
        hn = ops.rmsnorm(x, self.w.final_norm, c.rms_eps)
        logits = ops.gemm(hn, self.w.lm_head, out_dtype=torch.float32)
        idx, _ = ops.argmax_rows(logits)
        return idx, hn, logits



class VSMEngine(LlamaClipCore):
    # ------------------------------------------------------------------ heads
    def _mlp2(self, x, fc):
        h = ops.gemm(x, fc[0], bias=fc[1], epilogue=ops.EPI_RELU)
        return ops.gemm(h, fc[2], bias=fc[3])

    def _sam_attn(self, A, q, k, v, n, Nq, Nk, residual=None):
        """segment_anything Attention.forward: q [n*Nq,256], k/v [n*Nk,256] -> out_proj(attn) (+ residual)"""
        c = self.cfg
        qp = ops.gemm(q, A["wq"], bias=A["bq"])
        kp = ops.gemm(k, A["wk"], bias=A["bk"])
        vp = ops.gemm(v, A["wv"], bias=A["bv"])
        internal = qp.shape[1]
        hd = internal // c.sam_heads
        o = ops.attn_small(qp, kp, vp, n, c.sam_heads, Nq, Nk, hd, 1.0 / math.sqrt(hd))
        return ops.gemm(o, A["wo"], bias=A["bo"], residual=residual)

    def sam_low_res(self, fmap, seg_q, crop_of_loc):
        """fmap [B*g*g, C] OWL features, seg_q [n,256] seg queries, crop_of_loc list[int] -> low-res masks [n,4g,4g] fp32"""
        c, w = self.cfg, self.w
        g = c.owl_grid
        P = g * g
        n = seg_q.shape[0]
        D = c.sam_dim
        B = fmap.shape[0] // P
        img = ops.gemm(fmap, w.vp_w, bias=w.no_mask)                  # visual_projection + no_mask_embed (dense prompt)
        if crop_of_loc != list(range(B)):
            idx = self._const(("col", tuple(crop_of_loc)), crop_of_loc)
            img = img.view(B, P, D).index_select(0, idx).reshape(n * P, D).contiguous()
        keys = img
        tokens = torch.empty((n, 6, D), dtype=BF, device=self.dev)
        tokens[:, :5] = w.out_tokens
        tokens[:, 5] = seg_q
        tokens = tokens.view(n * 6, D)
        queries = tokens
        pe = w.dense_pe                                               # [P, D], broadcast over n
        for i, L in enumerate(w.sam_layers):
            if i == 0:
                queries = self._sam_attn(L["self_attn"], queries, queries, queries, n, 6, 6)
            else:
                q = ops.add_rows(queries, tokens)
                queries = self._sam_attn(L["self_attn"], q, q, queries, n, 6, 6, residual=queries)
            queries = ops.layernorm(queries, L["norm1"][0], L["norm1"][1], 1e-5)
            q = ops.add_rows(queries, tokens)
            k = ops.add_rows(keys, pe)
            queries = self._sam_attn(L["t2i"], q, k, keys, n, 6, P, residual=queries)
            queries = ops.layernorm(queries, L["norm2"][0], L["norm2"][1], 1e-5)
            h = ops.gemm(queries, L["w1"], bias=L["b1"], epilogue=ops.EPI_RELU)
            queries = ops.gemm(h, L["w2"], bias=L["b2"], residual=queries)
            queries = ops.layernorm(queries, L["norm3"][0], L["norm3"][1], 1e-5)
            q = ops.add_rows(queries, tokens)
            k = ops.add_rows(keys, pe)
            keys = self._sam_attn(L["i2t"], k, q, queries, n, P, 6, residual=keys)
            keys = ops.layernorm(keys, L["norm4"][0], L["norm4"][1], 1e-5)
        q = ops.add_rows(queries, tokens)
        k = ops.add_rows(keys, pe)
        queries = self._sam_attn(w.sam_final, q, k, keys, n, 6, P, residual=queries)
        queries = ops.layernorm(queries, w.sam_final_norm[0], w.sam_final_norm[1], 1e-5)
        mask_tok = queries.view(n, 6, D)[:, 1, :]                     # mask token 0 (row 0 is the IoU token)
        # upscaling: bilinear x2 -> conv3x3 -> LN2d -> GELU -> bilinear x2 -> conv3x3 -> GELU  (channels-last)
        u = ops.upsample2x_nhwc(keys, n, g, g, D)
        u = ops.gemm(ops.im2col3x3_nhwc(u, n, 2 * g, 2 * g, D), w.up0_w, bias=w.up0_b)
        u = ops.layernorm(u, w.up_ln[0], w.up_ln[1], 1e-6, act=ops.EPI_GELU)
        u = ops.upsample2x_nhwc(u, n, 2 * g, 2 * g, D // 4)
        u = ops.gemm(ops.im2col3x3_nhwc(u, n, 4 * g, 4 * g, D // 4), w.up1_w, bias=w.up1_b, epilogue=ops.EPI_GELU)
        hy = ops.gemm(mask_tok, w.hyper[0][0], bias=w.hyper[0][1], epilogue=ops.EPI_RELU)
        hy = ops.gemm(hy, w.hyper[1][0], bias=w.hyper[1][1], epilogue=ops.EPI_RELU)
        hy = ops.gemm(hy, w.hyper[2][0], bias=w.hyper[2][1])
        low = ops.mask_dot(u, hy.contiguous(), n, 16 * P, D // 8)
        return low.view(n, 4 * g, 4 * g)

    def owl_heads(self, fmap, det_q, crop_of_loc):
        """OwlViT.forward for n (crop, query) pairs -> logits [n,P], scores [n,P], boxes [n,P,4]"""
        c, w = self.cfg, self.w
        P = c.owl_grid ** 2
        B = fmap.shape[0] // P
        n = det_q.shape[0]
        Q = c.owl_query_dim
        y = ops.gemm(fmap, w.cls_w, bias=w.cls_b, out_dtype=torch.float32)      # [B*P, Q+2], shared by all queries of a crop
        hb = ops.gemm(fmap, w.box[0][0], bias=w.box[0][1], epilogue=ops.EPI_GELU)
        hb = ops.gemm(hb, w.box[1][0], bias=w.box[1][1], epilogue=ops.EPI_GELU)
        yb = ops.gemm(hb, w.box[2][0], bias=w.box[2][1], out_dtype=torch.float32)
        boxes = ops.owl_box_post(yb, w.box_bias, P, quant_bf16=self.heads_bf16).view(B, P, 4)
        if crop_of_loc == list(range(B)):
            logits, scores = ops.owl_class_post(y, det_q.contiguous(), P, Q, quant_bf16=self.heads_bf16)
            return logits.view(n, P), scores.view(n, P), boxes          # one entry per crop: boxes [n,P,4] with n == B
        idx = self._const(("col", tuple(crop_of_loc)), crop_of_loc)
        yy = y.view(B, P, Q + 2).index_select(0, idx).reshape(n * P, Q + 2).contiguous()
        logits, scores = ops.owl_class_post(yy, det_q.contiguous(), P, Q, quant_bf16=self.heads_bf16)
        return logits.view(n, P), scores.view(n, P), boxes.index_select(0, idx)

    # ------------------------------------------------------------------ whole-model entry points
    def model_forward(self, images, images_clip, input_ids, mode="detection"):
        """Teacher-forced single pass == VSMForCausalLM.model_forward(inference=True) (VSM.py:201-364), batched over B.
        input_ids [B,L] already contain the answer.  Returns dict of device tensors."""
        with ops.batch_invariant():
            return self._model_forward(images, images_clip, input_ids, mode)

    def _model_forward(self, images, images_clip, input_ids, mode):
        c = self.cfg
        B, L = input_ids.shape
        x, T, img_pos = self.prefill(input_ids, images_clip)
        ids_cpu = input_ids.cpu()
        rows, crop_of_loc = [], []
        for b in range(B):
            for k in (ids_cpu[b] == c.loc_token_idx).nonzero().flatten().tolist():
                assert k - 1 > img_pos, "[LOC] before the image is outside the reference's 255-offset hack (VSM.py:230-234)"
                rows.append(self.x_row(b, (k - 1) + c.clip_tokens - 1))
                crop_of_loc.append(b)
        if not rows:
            raise RuntimeError("no [LOC] token in input_ids: the reference fails here too (VSM.py:322 empty loop, visual_search.py:209-211)")
        out = self._heads(x, T, rows, crop_of_loc, images, mode)
        out["n_crops"], out["verified"] = B, [True] * B
        return out

    def _heads(self, x, T, rows, crop_of_loc, images, mode):
        c = self.cfg
        rows_t = self._const(("rows", tuple(rows)), rows)
        sel = ops.gather_rows(rows_t, x)
        hn = ops.rmsnorm(sel, self.w.final_norm, c.rms_eps)
        seg_q = self._mlp2(hn, self.w.fcs["seg"])
        det_q = self._mlp2(hn, self.w.fcs["det"])
        fmap = self.owl_feature_map(images)
        low = self.sam_low_res(fmap, seg_q, crop_of_loc)
        out = dict(hidden_loc=hn, seg_queries=seg_q, det_queries=det_q, feature_map=fmap, low_res_masks=low, crop_of_loc=crop_of_loc)
        if mode != "segmentation":
            out["pred_logits"], out["scores"], out["pred_boxes"] = self.owl_heads(fmap, det_q, crop_of_loc)
        return out

    def finish(self, out, am_host=None):
        """resolve a deferred inference(): the one host sync (greedy argmax of the answer rows vs the draft).  am_host: the
        argmax tensor already copied to the host by the caller (pipelined batches fetch it on a side stream)."""
        if out.get("verified") is None:
            am, draft, B = out.pop("_am"), out.pop("_draft"), out["n_crops"]
            am = (am_host if am_host is not None else am.cpu()).view(B, -1)
            ok = [bool((am[b] == draft).all()) for b in range(B)] if not out.pop("_forced") else [True] * B
            self.last_argmax = am
            self.stats["fallback"] += sum(1 for o in ok if not o)
            self.stats["verified"] += sum(1 for o in ok if o)
            out["verified"] = ok
        return out

    def inference(self, images, images_clip, prompt_ids, draft_ids, eos_token_id=2, max_new_tokens=100, mode="detection",
                  forced_ids=None, defer=False):
        """== VSMForCausalLM.inference (VSM.py:438-553) for a batch of crops sharing one prompt length.
        prompt_ids [B,Lp]; draft_ids [g] = the expected greedy answer incl. EOS (e.g. tokenizer("Sure, [LOC] .")+EOS).
        `forced_ids` (tests / synthetic weights only) forces the emitted tokens like a logits processor would, in which
        case verification compares nothing and the draft is taken as the answer.

        Runs in batch-invariant mode (ops.batch_invariant): a crop's outputs do not depend on the size of its batch."""
        with ops.batch_invariant():
            return self._inference(images, images_clip, prompt_ids, draft_ids, eos_token_id, max_new_tokens, mode, forced_ids, defer)

    def _inference(self, images, images_clip, prompt_ids, draft_ids, eos_token_id, max_new_tokens, mode, forced_ids, defer):
        c = self.cfg
        B, Lp = prompt_ids.shape
        g = len(draft_ids)
        draft = torch.as_tensor(draft_ids, dtype=torch.int64)
        ids = torch.cat([prompt_ids.cpu(), draft[:-1].unsqueeze(0).expand(B, -1)], dim=1).contiguous()      # host tensor
        key = self._graph_key(ids, B, Lp, draft_ids, mode) if defer else None
        if key is not None:
            dev = self._graph_run(key, images, images_clip, ids, Lp, g, mode)
        else:
            dev = self._crop_forward(images, images_clip, ids, None, Lp, g, mode)
        d_host = torch.as_tensor(draft_ids, dtype=torch.int64)
        out_ids = [torch.cat([prompt_ids[b].cpu(), d_host]) for b in range(B)]
        # crops whose greedy answer deviates from the draft are flagged (finish()); the caller re-runs them with exact
        # step-wise greedy decoding (VSMEngine.generate) so emitted ids are always the reference's greedy ids.  With
        # defer=True nothing here waits for the GPU: the caller can prepare the next chunk while this one runs.
        out = dict(dev)
        out.update(verified=None, _draft=d_host, _forced=forced_ids is not None, n_crops=B, output_ids=out_ids)
        return out if defer else self.finish(out)

    def _crop_forward(self, images, images_clip, ids, ids_dev, Lp, g, mode):
        """device work of one draft-verified batch: prefill over prompt + draft, logits of the g answer-predicting rows, heads.
        No host synchronisation and (once the shape has been seen) no host->device traffic: this is what a CUDA graph captures."""
        c = self.cfg
        B = ids.shape[0]
        x, T, img_pos = self.prefill(ids, images_clip, tail_rows=g, ids_dev=ids_dev)     # only the g answer-predicting rows are read below
        n_img = c.clip_tokens
        # rows that predict answer token j (j = 0..g-1): original index Lp-1+j -> spliced row +255
        pr = [self.x_row(b, (Lp - 1 + j) + n_img - 1) for b in range(B) for j in range(g)]
        hn, am, logits = self._logits_rows(x, self._const(("rows", tuple(pr)), pr))
        self.last_logits = logits.view(B, g, -1)
        out = dict(_am=am)
        if mode == "vqa":
            return out
        rows, crop_of_loc = [], []
        d_cpu = ids[0, Lp:].tolist() + [None]                 # draft[:-1] is in ids; the last draft token (EOS) predicts nothing
        for b in range(B):
            for j, tok in enumerate(d_cpu):
                if tok == c.loc_token_idx:
                    rows.append(self.x_row(b, (Lp - 1 + j) + n_img - 1))
                    crop_of_loc.append(b)
        if not rows:
            raise RuntimeError("no [LOC] token generated (reference: IndexError at visual_search.py:209-211)")
        out.update(self._heads(x, T, rows, crop_of_loc, images, mode))
        return out

    # ------------------------------------------------------------------ CUDA graphs for small frontier batches
    def _graph_key(self, ids, B, Lp, draft_ids, mode):
        """hashable shape key if this call can run as a captured graph: small batch, one <image>, the shared prefix already
        snapshotted and in use (steady state of a search), cache large enough"""
        if self.graph_max_batch <= 0 or B > self.graph_max_batch or self._capturing or not self.prefix_cache or self._prefix_ids is None \
                or ops.profiling:                 # (per-launch GEMM events of bench.py's roofline leg cannot be recorded inside a graph)
            return None
        pos = (ids[0] == IMAGE_TOKEN_INDEX).nonzero()
        if pos.numel() != 1:
            return None
        img_pos = int(pos[0, 0])
        P = len(self._prefix_ids)
        if img_pos - 1 != P or not bool((ids[:, :P] == torch.tensor(self._prefix_ids)).all()) or not bool((ids[:, img_pos] == IMAGE_TOKEN_INDEX).all()):
            return None
        return (B, Lp, img_pos, tuple(int(t) for t in draft_ids), mode, self.heads_bf16, self.tail_only)

    def _graph_run(self, key, images, images_clip, ids, Lp, g, mode):
        from . import _lib
        ent = self._graphs.get(key)
        B = ids.shape[0]
        P = len(self._prefix_ids)
        if ent is None:
            n = self._graph_seen.get(key, 0) + 1
            self._graph_seen[key] = n
            if n <= 2:                                        # eager warm-up: kernel attributes, device constants, cache, prefix rows
                return self._crop_forward(images, images_clip, ids, None, Lp, g, mode)
            ent = self._graph_capture(key, images, images_clip, ids, Lp, g, mode)
        if ent is False:                                      # capture failed once: stay eager for this shape
            return self._crop_forward(images, images_clip, ids, None, Lp, g, mode)
        ent["images"].copy_(images, non_blocking=True)
        ent["images_clip"].copy_(images_clip, non_blocking=True)
        ent["ids"].copy_(ids[:, P:], non_blocking=True)
        if self._prefix_slots < B:                            # slots that lost / never had the prefix rows
            self._cache[:, self._prefix_slots:B, :P].copy_(self._prefix_kv[:, None])
            self._prefix_slots = B
        ent["graph"].replay()
        _lib.launches += ent["launches"]
        self.stats["prefix_shared"] += B
        self.stats["graph_replays"] = self.stats.get("graph_replays", 0) + 1
        self._P, self._Tn = ent["P"], ent["Tn"]
        # the graph's output buffers are overwritten by its next replay: hand out copies of what callers keep
        out = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in ent["out"].items()}
        self.last_logits = None
        return out

    def _graph_capture(self, key, images, images_clip, ids, Lp, g, mode):
        from . import _lib
        B = ids.shape[0]
        P = len(self._prefix_ids)
        if len(self._graphs) >= 16:
            self._graphs.pop(next(iter(self._graphs)))
        try:
            st_images, st_clip = torch.empty_like(images), torch.empty_like(images_clip)
            st_ids = ids[:, P:].contiguous().to(self.dev)
            st_images.copy_(images)
            st_clip.copy_(images_clip)
            if self._prefix_slots < B:
                self._cache[:, self._prefix_slots:B, :P].copy_(self._prefix_kv[:, None])
                self._prefix_slots = B
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            l0 = _lib.launches
            shared0 = self.stats["prefix_shared"]
            self._capturing = True
            try:
                with torch.cuda.graph(graph):
                    out = self._crop_forward(st_images, st_clip, ids, st_ids, Lp, g, mode)
            finally:
                self._capturing = False
            self.stats["prefix_shared"] = shared0
            keep = ("_am", "low_res_masks", "pred_logits", "scores", "pred_boxes", "crop_of_loc")
            ent = dict(graph=graph, images=st_images, images_clip=st_clip, ids=st_ids, launches=_lib.launches - l0, P=self._P, Tn=self._Tn,
                       out={k: v for k, v in out.items() if k in keep})
            _lib.launches = l0
            self.stats["graphs_captured"] = self.stats.get("graphs_captured", 0) + 1
        except Exception as e:          # never let a capture problem break the search: this shape stays on the eager path
            self._capturing = False
            self.stats["graph_capture_errors"] = self.stats.get("graph_capture_errors", 0) + 1
            self.last_graph_error = repr(e)
            ent = False
        self._graphs[key] = ent
        return ent

    def generate_many(self, prompt_ids, images_clip, max_new_tokens=100, eos_token_id=2):
        """Exact greedy decoding for B crops that share one prompt LENGTH (the cue question of the weak-cue branch asked of many
        crops, visual_search.py:427-431): ONE batched prefill, then one decode step per token for the whole batch (every weight
        byte read once for B tokens); sequences that have emitted EOS keep stepping and are ignored.
        -> list of B token-id lists (prompt + answer incl. EOS), like `generate` gives for one crop."""
        c = self.cfg
        B, L = prompt_ids.shape
        room = self.MAX_POSITIONS - (L - 1 + c.clip_tokens)
        x, T, img_pos = self.prefill(prompt_ids.cpu(), images_clip, reserve=max(0, min(max_new_tokens, room)))
        last = self._const(("rows", tuple(self.x_row(b, T - 1) for b in range(B))), [self.x_row(b, T - 1) for b in range(B)])
        hn, am, logits = self._logits_rows(x, last)
        outs = [prompt_ids[b].cpu().tolist() for b in range(B)]
        done = [False] * B
        past = T
        for step in range(max_new_tokens):
            nxt = am.cpu().tolist()                       # one D2H per step for the whole batch
            for b in range(B):
                if not done[b]:
                    outs[b].append(int(nxt[b]))
                    done[b] = int(nxt[b]) == eos_token_id
            if all(done) or step == max_new_tokens - 1:
                break
            am, hn, logits = self.decode_step(torch.tensor(nxt, dtype=torch.int64, device=self.dev), B, past)
            past += 1
        return outs

    def generate(self, prompt_ids, images_clip, max_new_tokens=100, eos_token_id=2, forced_ids=None):
        """Exact greedy decoding for ONE sequence on the fused-QKV cache (reference: HF generate, use_cache=False —
        mathematically the same sequence).  Returns (output_ids list, per-step argmax list, residual rows)."""
        c = self.cfg
        assert prompt_ids.shape[0] == 1
        L = prompt_ids.shape[1]
        room = self.MAX_POSITIONS - (L - 1 + c.clip_tokens)
        x, T, img_pos = self.prefill(prompt_ids.to(self.dev), images_clip, reserve=max(0, min(max_new_tokens, room)))
        last = torch.tensor([self.x_row(0, T - 1)], dtype=torch.int64, device=self.dev)
        hn, am, logits = self._logits_rows(x, last)
        out = prompt_ids[0].cpu().tolist()
        argmaxes = []
        past = T
        for step in range(max_new_tokens):
            nxt = int(am[0])
            argmaxes.append(nxt)
            if forced_ids is not None and step < len(forced_ids):
                nxt = int(forced_ids[step])
            out.append(nxt)
            if nxt == eos_token_id or step == max_new_tokens - 1:
                break
            am, hn, logits = self.decode_step(torch.tensor([nxt], dtype=torch.int64, device=self.dev), 1, past)
            past += 1
        return out, argmaxes
