"""SEAL VQA LLM on the sm_90a kernels — the model that brackets the visual search in `vstar_bench_eval.py`
(SURVEY.md §8 rows a18-a20, §8f-1).

  VQAWeights / VQAEngine : LlavaSearchLlamaForCausalLM (/root/reference/LLaVA/llava/model/language_model/llava_search_llama.py:56-141,
                           llava_search_arch.py:83-279): CLIP-L -> BOTH projectors (linear "long" 256 tokens; LayerNorm ->
                           PerceiverResampler(depth 6, 16 heads x 96, 32 latents) -> Linear "short" 32 tokens), <image>/<object>
                           splicing with the long/short switches, Llama prefill / greedy decode on the fused-QKV cache, option
                           scoring with the question prefix kept in the cache (vstar_bench_eval.py:116-165).
  VQA_LLM                : drop-in mirror of `vstar_bench_eval.VQA_LLM` (free_form_inference, multiple_choices_inference,
                           get_patch, get_object_crop).

The reference runs this model in fp16 (LLaVA/llava/model/builder.py:43).  The engine runs in bf16 by default (fp32
accumulation; tolerance stated in tests/test_vqa_gpu.py) or, opt-in, in fp16 like the reference on the _f16 variants of the
same kernels: VQAWeights(..., dtype=torch.float16), load_pretrained_model(..., torch_dtype=torch.float16) or
VQA_LLM(args) with args.vqa_dtype = "fp16".  fp16 brings the option NLLs and logits close to the reference's own
numbers (tests/test_vqa_fp16_gpu.py; DESIGN.md §7b).  The VSM stays bf16, as in the reference.
free_form_inference(temperature > 0, top_p) samples like the reference's `generate(do_sample=True)`: one vsb_sample_rows_f32
launch per decode step in place of the greedy argmax (oracle/sampling_oracle.py; DESIGN.md §7b).
free_form_inference(num_beams = k) runs HF's beam search (transformers 4.31): VQAEngine.beam_search, one vsb_beam_candidates_f32
launch per step and copy-on-fork KV-row copies (vstar_b200/beam.py, oracle/beam_oracle.py; DESIGN.md §7b).
DecodeStream.admit takes the same settings per request, so one decode stream mixes greedy, sampled and beam requests
(vsb_sample_rows_var_f32, vsb_copy_slot_rows_b16; DESIGN.md §7b).
"""
from __future__ import annotations

from collections import namedtuple

import numpy as np
import torch

from . import ops
from .beam import DEFAULT_EARLY_STOPPING, DEFAULT_LENGTH_PENALTY, BeamRequest, check_beams, fork_slots
from .config import VSMConfig
from .engine import CoreWeights, LlamaClipCore
from .kv_pages import PAGE_ROWS, GrowingPool, PagePool, pages_for, plan_chunks
from .vsm import CLIP_MEAN, SyntheticTokenizer, _normalize_into

BF = torch.bfloat16
VQA_DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}
IMAGE_TOKEN_INDEX = -200
OBJECT_TOKEN_INDEX = -300
DEFAULT_IMAGE_TOKEN = "<image>"
DEFAULT_OBJECT_TOKEN = "<object>"

DEFAULT_TOP_K = 50        # transformers 4.31 GenerationConfig.top_k, used unless the checkpoint's generation_config.json sets it

VICUNA_V1_SYSTEM = ("A chat between a curious user and an artificial intelligence assistant. "
                    "The assistant gives helpful, detailed, and polite answers to the user's questions.")


def build_prompt_v1(question_with_image_token, answer=None):
    """conv_templates['v1'] (LLaVA/llava/conversation.py:252-262; SeparatorStyle.TWO, sep ' ', sep2 '</s>')"""
    ret = VICUNA_V1_SYSTEM + " " + "USER: " + question_with_image_token + " "
    if answer:
        ret += "ASSISTANT: " + answer + "</s>"
    else:
        ret += "ASSISTANT:"
    return ret


def tokenizer_image_object_token(prompt, tokenizer, image_token_index=IMAGE_TOKEN_INDEX, object_token_index=OBJECT_TOKEN_INDEX):
    """LLaVA/llava/mm_utils.py:65-87 (behaviour kept verbatim: defines the token sequence)"""
    prompt_chunks = []
    for prompt_chunk in prompt.split("<image>"):
        prompt_chunks.extend(prompt_chunk.split("<object>"))
    prompt_chunks = [tokenizer(chunk).input_ids for chunk in prompt_chunks]

    def insert_separator(X, seps):
        return [ele for sublist in zip(X, seps) for ele in sublist][:-1]

    input_ids = []
    offset = 0
    if len(prompt_chunks) > 0 and len(prompt_chunks[0]) > 0 and prompt_chunks[0][0] == tokenizer.bos_token_id:
        offset = 1
        input_ids.append(prompt_chunks[0][0])
    sep = [[image_token_index] * (offset + 1)] + [[object_token_index] * (offset + 1)] * (len(prompt_chunks) - 1)
    for x in insert_separator(prompt_chunks, sep):
        input_ids.extend(x[offset:])
    return input_ids


def check_sampling(top_k, top_p):
    """the arguments the reference's warpers validate (TopKLogitsWarper / TopPLogitsWarper) -> (top_k, top_p) for the sampler:
    top_k None or 0 = no top-k filter, top_p None = no nucleus filter"""
    top_k = 0 if top_k is None else top_k
    if isinstance(top_k, bool) or not isinstance(top_k, int) or top_k < 0:
        raise ValueError(f"`top_k` has to be a non-negative integer, but is {top_k!r}")
    if top_p is not None:
        top_p = float(top_p)
        if not (0.0 <= top_p <= 1.0):
            raise ValueError(f"`top_p` has to be a float >= 0 and <= 1, but is {top_p}")
    return top_k, top_p


def draw_seeds(n):
    """n sampler seeds from torch's default generator, one int64 draw per request in request order (where HF's `sample()`
    takes its randomness for torch.multinomial), so torch.manual_seed(s) reproduces a sampled call"""
    return torch.empty(n, dtype=torch.int64).random_().tolist()


def generation_top_k(model_path, beams=False):
    """top_k of the checkpoint's generation_config.json, else the transformers 4.31 default (50).
    beams=True: -> (top_k, length_penalty, early_stopping), each from the file when it sets it, else the 4.31 default
    (50, 1.0, False)"""
    import json
    import os
    path = os.path.join(str(model_path), "generation_config.json")
    cfg = {}
    if os.path.isfile(path):
        with open(path) as f:
            cfg = json.load(f)
    k = cfg.get("top_k")
    k = DEFAULT_TOP_K if k is None else int(k)
    if not beams:
        return k
    lp = cfg.get("length_penalty")
    es = cfg.get("early_stopping")
    return k, DEFAULT_LENGTH_PENALTY if lp is None else float(lp), DEFAULT_EARLY_STOPPING if es is None else es


class VQAWeights(CoreWeights):
    """CoreWeights + the object projector `model.mm_projector_object.{0,1,2}` (multimodal_projector/builder.py:54-68).
    dtype: torch.bfloat16 (default) or torch.float16 (the reference's dtype for this model)."""

    def __init__(self, cfg: VSMConfig, get, device="cuda", dtype=BF, quant=None):
        super().__init__(cfg, get, device, dtype=dtype, quant=quant)
        g, lin = self._g, self._lin
        p = "model.mm_projector_object."
        self.pj_ln = (g(p + "0.weight"), g(p + "0.bias"))
        self.latents = g(p + "1.latents")
        self.media_pos = g(p + "1.media_pos_emb").reshape(1, -1).contiguous()
        self.pj_layers = []
        for i in range(6):
            a, f = f"{p}1.layers.{i}.0.", f"{p}1.layers.{i}.1."
            self.pj_layers.append(dict(
                nm=(g(a + "norm_media.weight"), g(a + "norm_media.bias")), nl=(g(a + "norm_latents.weight"), g(a + "norm_latents.bias")),
                wq=lin(a + "to_q.weight"), wkv=lin(a + "to_kv.weight"), wo=lin(a + "to_out.weight"),
                ffn=(g(f + "0.weight"), g(f + "0.bias")), w1=lin(f + "1.weight"), w2=lin(f + "3.weight")))
        self.pj_norm = (g(p + "1.norm.weight"), g(p + "1.norm.bias"))
        self.pj_out = (lin(p + "2.weight"), g(p + "2.bias"))

    def linear_bytes(self):
        nb = ops.weight_nbytes
        return super().linear_bytes() + sum(nb(L[k]) for L in self.pj_layers for k in ("wq", "wkv", "wo", "w1", "w2")) + nb(self.pj_out[0])


class VQAEngine(LlamaClipCore):
    HEADS, DHEAD, NLAT = 16, 96, 32

    def __init__(self, weights: VQAWeights, max_tokens=1536):
        super().__init__(weights, max_tokens=max_tokens)

    # ------------------------------------------------------------------ projectors
    def project_both(self, pixels):
        """encode_images / project_features (llava_search_arch.py:83-93): pixels [n,3,224,224] in the engine dtype ->
        (long [n*256, d], short [n*32, d])"""
        c, w = self.cfg, self.w
        n = pixels.shape[0]
        ct, S = self.clip_tokens(pixels)                                   # [n*257, C] incl. CLS
        P = S - 1
        rows = torch.arange(n * S, device=self.dev).view(n, S)[:, 1:].reshape(-1).contiguous()
        feats = ops.gather_rows(rows, ct)                                  # hidden_states[-2][:, 1:]
        long_ = ops.gemm(feats, w.mm_w, bias=w.mm_b)
        C = feats.shape[1]
        inner = self.HEADS * self.DHEAD
        x = ops.layernorm(feats, w.pj_ln[0], w.pj_ln[1], 1e-5)
        x = ops.add_rows(x, w.media_pos)                                   # + media_pos_emb[:1]
        lat = w.latents.repeat(n, 1).contiguous()                          # [n*32, C]
        NK = P + self.NLAT
        kv = torch.empty((n * NK, 2 * inner), dtype=self.dtype, device=self.dev)
        for L in w.pj_layers:
            xm = ops.layernorm(x, L["nm"][0], L["nm"][1], 1e-5)
            lt = ops.layernorm(lat, L["nl"][0], L["nl"][1], 1e-5)
            q = ops.gemm(lt, L["wq"])
            # to_kv(cat(media, latents)): two GEMMs scatter their rows into one [n, P+32, 2*inner] buffer
            ops.gemm(xm, L["wkv"], out=kv, rows_per_group=P, group_stride=NK, group_offset=0)
            ops.gemm(lt, L["wkv"], out=kv, rows_per_group=self.NLAT, group_stride=NK, group_offset=P)
            o = ops.attn_small(q, kv[:, :inner], kv[:, inner:], n, self.HEADS, self.NLAT, NK, self.DHEAD, self.DHEAD ** -0.5)
            lat = ops.gemm(o, L["wo"], residual=lat)
            h = ops.layernorm(lat, L["ffn"][0], L["ffn"][1], 1e-5)
            h = ops.gemm(h, L["w1"], epilogue=ops.EPI_GELU)
            lat = ops.gemm(h, L["w2"], residual=lat)
        res = ops.layernorm(lat, w.pj_norm[0], w.pj_norm[1], 1e-5)
        short = ops.gemm(res, w.pj_out[0], bias=w.pj_out[1])
        return long_, short

    # ------------------------------------------------------------------ splice (llava_search_arch.py:139-216)
    def build_embeds(self, input_ids, image, object_crops=None, images_long=None, objects_long=None):
        """input_ids: python list with one -200 and k -300 placeholders -> embeds [T, d] on the device"""
        return self.build_embeds_batch([(input_ids, image, object_crops, images_long, objects_long)])[0]

    def _splice(self, ids, img_long, img_short, obj_long, obj_short, images_long, objects_long):
        c = self.cfg
        segs = []                                   # ("ids", list) | ("feat", tensor [m,d])
        s = ids.index(IMAGE_TOKEN_INDEX)
        use_long = images_long is None or bool(images_long[0])
        segs += [("ids", ids[:s]), ("feat", img_long if use_long else img_short)]
        cur = ids[s + 1:]
        oi = 0
        while OBJECT_TOKEN_INDEX in cur:
            s = cur.index(OBJECT_TOKEN_INDEX)
            short = objects_long is None or not bool(objects_long[oi])
            f = obj_short[oi * 32:(oi + 1) * 32] if short else obj_long[oi * c.clip_tokens:(oi + 1) * c.clip_tokens]
            segs += [("ids", cur[:s]), ("feat", f)]
            oi += 1
            cur = cur[s + 1:]
        if cur:
            segs.append(("ids", cur))
        T = sum(len(v) if k == "ids" else v.shape[0] for k, v in segs)
        x = torch.empty((T, c.hidden), dtype=self.dtype, device=self.dev)
        t = 0
        for k, v in segs:
            n = len(v) if k == "ids" else v.shape[0]
            if n == 0:
                continue
            if k == "ids":
                ops.gather_rows(torch.tensor(v, dtype=torch.int64, device=self.dev), self.w.embed, out=x[t:t + n])
            else:
                ops.copy2d(v, x[t:t + n])
            t += n
        return x

    # ------------------------------------------------------------------ LM
    def prefill_embeds(self, x, reserve=0):
        """x [T,d] (consumed in place) -> residual stream after all layers; cache positions 0..T.  reserve: positions the
        caller will append (the slot is sized for T + reserve; beyond the 2048 RoPE rows raises VsbError)"""
        T = x.shape[0]
        self._ensure_cache(1, self._capacity(T + reserve))
        self._prefix_slots = 0
        self._llm_layers(x, 1, T, 0)
        self.kv_epoch = getattr(self, "kv_epoch", 0) + 1        # handles to an older prefix are stale from here on
        return x

    def append_tokens(self, tokens, past):
        """run `tokens` (python list) on top of `past` cached positions -> logits fp32 [n, V] for every new position"""
        ids = torch.tensor(tokens, dtype=torch.int64, device=self.dev)
        x = ops.gather_rows(ids, self.w.embed)
        if past + len(tokens) > self._cache_shape[2]:
            self._ensure_cache(self._cache_shape[1], self._capacity(past + len(tokens) + 64), keep=True)
        self._llm_layers(x, 1, len(tokens), past)
        hn = ops.rmsnorm(x, self.w.final_norm, self.cfg.rms_eps)
        return ops.gemm(hn, self.w.lm_head, out_dtype=torch.float32)

    def last_logits(self, x):
        rows = torch.tensor([x.shape[0] - 1], dtype=torch.int64, device=self.dev)
        hn, am, logits = self._logits_rows(x, rows)
        return logits

    def _sampler(self, temperature, top_k, top_p, seeds):
        """None for greedy decoding (temperature None or <= 0); else fn(logits [B, V], step) -> int32 [B] tokens drawn by
        vsb_sample_rows_f32 with one seed per row (uploaded once per call; None: one default-generator draw for a single row)"""
        if temperature is None or not temperature > 0:
            return None
        top_k, top_p = check_sampling(top_k, top_p)
        seeds = draw_seeds(1) if seeds is None else seeds
        sd = torch.tensor([_signed64(s) for s in seeds], dtype=torch.int64, device=self.dev)
        T, dtype = float(temperature), self.dtype
        return lambda logits, step: ops.sample_rows(logits, T, top_k, top_p, dtype, sd, step)

    def generate(self, input_ids, image, object_crops=None, images_long=None, objects_long=None, max_new_tokens=200, eos_token_id=2,
                 stop_ids=None, stop_fn=None, temperature=0, top_k=DEFAULT_TOP_K, top_p=None, seed=None, num_beams=1,
                 length_penalty=DEFAULT_LENGTH_PENALTY, early_stopping=DEFAULT_EARLY_STOPPING):
        """greedy `model.generate(use_cache=True, do_sample=False)` (vstar_bench_eval.py:91-103) -> list of new token ids.
        stop_ids: stop once the output ends with these ids; stop_fn(new_ids) -> bool: HF-style stopping criterion.
        temperature > 0: sampled decoding instead (`do_sample=True` with top_k / top_p, ops.sample_rows); token t is drawn with
        (seed, step t), seed None = one draw from torch's default generator.
        num_beams > 1: beam search (beam_search; its chosen hypothesis' ids), stop_ids at most [eos_token_id], stop_fn then
        receives the k running beams' new ids."""
        if self._beam_args(num_beams, temperature, stop_ids, eos_token_id, early_stopping):
            return self.beam_search([(input_ids, image, object_crops, images_long, objects_long)], num_beams, max_new_tokens,
                                    eos_token_id, length_penalty, early_stopping, stop_fn)[0][0]
        sampler = self._sampler(temperature, top_k, top_p, None if seed is None else [seed])
        x = self.build_embeds(input_ids, image, object_crops, images_long, objects_long)
        T = x.shape[0]
        self.prefill_embeds(x, reserve=max(0, min(max_new_tokens, self.MAX_POSITIONS - T)))
        logits = self.last_logits(x)
        out = []
        past = T
        for step in range(max_new_tokens):
            nxt = int(ops.argmax_rows(logits)[0][0] if sampler is None else sampler(logits, step)[0])
            out.append(nxt)
            if nxt == eos_token_id or (stop_ids and out[-len(stop_ids):] == list(stop_ids)) or \
                    (stop_fn is not None and stop_fn(out)):
                break
            logits = self.append_tokens([nxt], past)
            past += 1
        return out

    # ------------------------------------------------------------------ continuous-batched greedy decode (SURVEY.md §8f-1)
    def prefill_ragged(self, xs, reserve=0, slots=0):
        """xs: list of [T_b, d] input embeddings (consumed).  Sequences are LEFT-padded in the shared cache: sequence b
        occupies cache rows [Tpad - T_b, Tpad) of batch slot b, so every sequence ends at the same row and one decode
        step is ONE set of kernels for the whole batch (each weight byte read once for B tokens).  Runs of neighbouring
        sequences of EQUAL length are prefilled as one batch (M = G * T rows) - generate_batch orders its requests by length.
        slots: cache slots to hold (at least B; beam search keeps its other beams on slots B..).
        -> (last-position logits fp32 [B, V], Tpad, lengths)"""
        B = len(xs)
        lens = [int(x.shape[0]) for x in xs]
        Tpad = max(lens)
        self._ensure_cache(max(B, slots), self._capacity(Tpad + reserve))
        self._prefix_slots = 0
        Tm = self._cache_shape[2]
        last = []
        b = 0
        while b < B:
            G = 1
            while b + G < B and lens[b + G] == lens[b]:
                G += 1
            T = lens[b]
            x = torch.cat(xs[b:b + G], 0).contiguous() if G > 1 else xs[b]
            self._llm_layers(x, G, T, 0, cache_row_offset=b * Tm + (Tpad - T))
            last += [x[g * T + T - 1:g * T + T] for g in range(G)]
            b += G
        self.kv_epoch = getattr(self, "kv_epoch", 0) + 1
        hn = ops.rmsnorm(torch.cat(last, 0).contiguous(), self.w.final_norm, self.cfg.rms_eps)
        return ops.gemm(hn, self.w.lm_head, out_dtype=torch.float32), Tpad, lens

    def decode_ragged(self, tokens, lens, Tpad, step):
        """one decode step for the left-padded batch: tokens int64 [B] (token `step` of every answer) -> logits fp32 [B, V]"""
        B = len(lens)
        ids = torch.as_tensor(tokens, dtype=torch.int64, device=self.dev)
        x = ops.gather_rows(ids, self.w.embed)
        if Tpad + step + 1 > self._cache_shape[2]:
            self._ensure_cache(self._cache_shape[1], self._capacity(Tpad + step + 64), keep=True)
        positions = torch.tensor([n + step for n in lens], dtype=torch.int32, device=self.dev)
        k_start = torch.tensor([Tpad - n for n in lens], dtype=torch.int32, device=self.dev)
        self._llm_layers(x, B, 1, Tpad + step, positions=positions, k_start=k_start)
        hn = ops.rmsnorm(x, self.w.final_norm, self.cfg.rms_eps)
        return ops.gemm(hn, self.w.lm_head, out_dtype=torch.float32)

    def generate_batch(self, requests, max_new_tokens=200, eos_token_id=2, stop_ids=None, temperature=0, top_k=DEFAULT_TOP_K, top_p=None,
                       seeds=None, num_beams=1, length_penalty=DEFAULT_LENGTH_PENALTY, early_stopping=DEFAULT_EARLY_STOPPING):
        """greedy generation for several (input_ids, image, object_crops, images_long, objects_long) requests at once.
        Same per-sequence semantics as generate(); finished sequences idle (their slots keep stepping, results ignored).
        temperature > 0: sampled decoding as in generate(), request i with seeds[i] (None = one default-generator draw per
        request, in request order).  num_beams > 1: beam search as in generate(), every request on its own k slots.
        -> list of new-token lists"""
        if self._beam_args(num_beams, temperature, stop_ids, eos_token_id, early_stopping):
            return [ids for ids, _ in self.beam_search(requests, num_beams, max_new_tokens, eos_token_id, length_penalty, early_stopping)]
        if temperature is not None and temperature > 0 and seeds is None:
            seeds = draw_seeds(len(requests))
        xs = self.build_embeds_batch(list(requests))           # one CLIP + projector pass for every image of the batch
        perm = sorted(range(len(xs)), key=lambda i: int(xs[i].shape[0]))       # equal lengths next to each other (stable)
        xs = [xs[i] for i in perm]
        sampler = self._sampler(temperature, top_k, top_p, None if seeds is None else [seeds[i] for i in perm])
        longest = max(int(x.shape[0]) for x in xs)
        logits, Tpad, lens = self.prefill_ragged(xs, reserve=max(0, min(max_new_tokens, self.MAX_POSITIONS - longest)))
        B = len(xs)
        outs = [[] for _ in range(B)]
        done = [False] * B
        for step in range(max_new_tokens):
            nxt = (ops.argmax_rows(logits)[0] if sampler is None else sampler(logits, step)).tolist()   # one D2H per step
            for b in range(B):
                if done[b]:
                    continue
                outs[b].append(int(nxt[b]))
                if nxt[b] == eos_token_id or (stop_ids and outs[b][-len(stop_ids):] == list(stop_ids)):
                    done[b] = True
            if all(done) or step == max_new_tokens - 1:
                break
            logits = self.decode_ragged(nxt, lens, Tpad, step)
        res = [None] * B
        for k, i in enumerate(perm):
            res[i] = outs[k]
        return res

    def decode_stream(self, max_slots, max_positions=None, eos_token_id=2, temperature=0, num_beams=1, kv_pages=None, kv_swap_pages=None,
                      prefill_chunk=None):
        """Decode batch that admits a request whenever a slot is free (DecodeStream).  max_positions: cache rows per slot
        (default self.max_tokens); a request's prompt plus its max_new_tokens must fit in them.  kv_pages = N: the KV cache
        is a pool of N pages of kv_pages.PAGE_ROWS rows and a request reserves only the pages it needs (DecodeStream); None
        keeps one cache slot of max_positions rows per decode row.  kv_swap_pages = M (with kv_pages): requests take pages as
        they write them and are preempted to a pinned host swap area of M pages when the pool runs dry.  prefill_chunk = C (with
        kv_pages, without kv_swap_pages): admitted prompts are prefilled C rows per step alongside the running requests' decode
        rows (DecodeStream).  Generation settings belong to
        each request: DecodeStream.admit(..., temperature=, top_k=, top_p=, seed=, num_beams=, ...) samples or beam-searches
        it; the stream-wide temperature > 0 and num_beams > 1 are refused, since every sampled request needs its own seed."""
        if temperature is not None and temperature > 0:
            raise NotImplementedError("decode_stream takes no stream-wide temperature: sample a request with "
                                      "DecodeStream.admit(..., temperature=, top_k=, top_p=, seed=)")
        if num_beams != 1:
            raise NotImplementedError("decode_stream takes no stream-wide num_beams: beam-search a request with "
                                      "DecodeStream.admit(..., num_beams=, length_penalty=, early_stopping=)")
        return DecodeStream(self, max_slots, self.max_tokens if max_positions is None else max_positions, eos_token_id, kv_pages=kv_pages,
                            kv_swap_pages=kv_swap_pages, prefill_chunk=prefill_chunk)

    def spliced_length(self, input_ids, n_crops=0, images_long=None, objects_long=None):
        """rows the spliced sequence of build_embeds(input_ids, ...) has, computed on the host (the rule of _splice)"""
        ids = list(input_ids)
        n_obj = ids.count(OBJECT_TOKEN_INDEX)
        if ids.count(IMAGE_TOKEN_INDEX) != 1 or n_obj > n_crops:
            raise ValueError(f"a request needs one image token and at most {n_crops} object tokens (one per crop), got "
                             f"{ids.count(IMAGE_TOKEN_INDEX)} and {n_obj}")
        long_img = images_long is None or bool(images_long[0])
        T = len(ids) - 1 - n_obj + (self.cfg.clip_tokens if long_img else self.NLAT)
        for oi in range(n_obj):
            short = objects_long is None or not bool(objects_long[oi])
            T += self.NLAT if short else self.cfg.clip_tokens
        return T

    def _beam_args(self, num_beams, temperature, stop_ids, eos_token_id, early_stopping):
        """True when the call runs beam search (num_beams > 1); raises on the combinations beam search does not serve"""
        check_beams(num_beams, early_stopping)
        if num_beams == 1:
            return False
        if temperature is not None and temperature > 0:
            raise NotImplementedError("num_beams > 1 with temperature > 0 (HF beam_sample) is not implemented")
        if stop_ids and list(stop_ids) != [eos_token_id]:
            raise ValueError(f"with num_beams > 1 the only stop sequence is eos ([{eos_token_id}]), got {list(stop_ids)}")
        return True

    def beam_search(self, requests, num_beams, max_new_tokens=200, eos_token_id=2, length_penalty=DEFAULT_LENGTH_PENALTY,
                    early_stopping=DEFAULT_EARLY_STOPPING, stop_fn=None, on_step=None):
        """HF `beam_search` (transformers 4.31, one returned sequence) for several (input_ids, image, object_crops, images_long,
        objects_long) requests at once -> [(new token ids, score of the chosen hypothesis)], the ids as the reference's
        generate(num_beams=k) returns them after the prompt (the hypothesis, then eos if it is shorter than max_length).

        Request r is prefilled once (left-padded as in generate_batch) and its prompt rows are copied to its k - 1 other cache
        slots; every step then decodes all R * k slots in one decode_ragged call.  One vsb_beam_candidates_f32 launch selects
        each request's 2k candidates, one copy brings them to the host, and vstar_b200.beam applies the scorer.  Beams move by
        copy-on-fork: a surviving parent keeps its slot for its first child, later children take the slots of beams that died
        and get the parent's generated rows [Tpad, Tpad + step) by one vsb_copy_cache_rows_b16 launch, so no launch reads a
        slot it writes.  stop_fn(running beams' new ids, k lists in beam order) -> bool ends the search (HF stopping
        criteria, called after every step); requests that are done idle.  on_step(step, logits, slots, beams): observes every
        step's logits fp32 [*, V] with, per request in order of length, its beams' logits rows and new ids (tests replay it)."""
        check_beams(num_beams, early_stopping)
        k = num_beams
        dev = self.dev
        xs = self.build_embeds_batch(list(requests))
        perm = sorted(range(len(xs)), key=lambda i: int(xs[i].shape[0]))
        xs = [xs[i] for i in perm]
        R = len(xs)
        reqs = [BeamRequest(k, len(requests[i][0]), max_new_tokens, eos_token_id, length_penalty, early_stopping) for i in perm]
        longest = max(int(x.shape[0]) for x in xs)
        logits, Tpad, lens = self.prefill_ragged(xs, reserve=max(0, min(max_new_tokens, self.MAX_POSITIONS - longest)), slots=R * k)
        # request r: beam 0 on slot r (prefilled), slots R + r*(k-1) .. for its other beams
        owned = [[r] + [R + r * (k - 1) + j for j in range(k - 1)] for r in range(R)]
        if k > 1:
            ops.copy_cache_rows(self._cache, [(r, s) for r in range(R) for s in owned[r][1:]], 0, Tpad)
        slot_lens = [0] * (R * k)
        for r in range(R):
            for s in owned[r]:
                slot_lens[s] = lens[r]
        beam_slot = [[r] for r in range(R)]                 # logical beam -> cache slot (logits row) per request
        tokens = [0] * (R * k)
        host = torch.empty(2 * R * k, dtype=torch.int32).pin_memory()
        cand = torch.empty((3, R, 2 * k), dtype=torch.int32, device=dev)
        for step in range(max_new_tokens):
            k_in = len(beam_slot[0])
            n = R * k_in
            host[:n] = torch.tensor([s for bs in beam_slot for s in bs], dtype=torch.int32)
            host[n:2 * n].view(torch.float32)[:] = torch.tensor([x for q in reqs for x in q.scores], dtype=torch.float32)
            if on_step is not None:
                on_step(step, logits, [list(bs) for bs in beam_slot], [[list(b) for b in q.beams] for q in reqs])
            up = host[:2 * n].to(dev, non_blocking=True)
            ops.beam_candidates(logits, up[:n].view(R, k_in), up[n:].view(torch.float32).view(R, k_in), k, self.dtype, out=cand)
            c = cand.cpu()                                  # the one device-to-host copy of the step
            sc, tok, bm = c[0].view(torch.float32).tolist(), c[1].tolist(), c[2].tolist()
            pairs = []
            for r, q in enumerate(reqs):
                if q.done:
                    continue
                nxt = q.process(list(zip(sc[r], tok[r], bm[r])))
                new, forks = fork_slots(beam_slot[r], nxt, owned[r])
                pairs += forks
                for s, (_, t, _) in zip(new, nxt):
                    tokens[s] = t
                beam_slot[r] = new
            if all(q.done for q in reqs) or step == max_new_tokens - 1:
                break
            if stop_fn is not None and any(not q.done and stop_fn([list(b) for b in q.beams]) for q in reqs):
                break
            if pairs and step > 0:
                ops.copy_cache_rows(self._cache, pairs, Tpad, Tpad + step)
            logits = self.decode_ragged(tokens, slot_lens, Tpad, step)
        res = [None] * R
        for r, i in enumerate(perm):
            res[i] = reqs[r].finalize()
        return res

    def option_losses(self, question_ids, options_ids, image, object_crops=None, images_long=None, objects_long=None):
        """multiple_choices_inference core (vstar_bench_eval.py:127-163).  Returns (losses fp32 [n_options] on host, argmin)."""
        return self.option_losses_batch([(question_ids, options_ids, image, object_crops, images_long, objects_long)])[0]

    def build_embeds_batch(self, items):
        """items: [(input_ids, image [1,3,224,224], object_crops [k,3,224,224] | None, images_long, objects_long)] -> list of
        embeds [T_i, d].  ONE CLIP + projector pass over every image and object crop of the batch."""
        c = self.cfg
        pix, spans = [], []
        for ids, image, crops, il, ol in items:
            k = 0 if crops is None else int(crops.shape[0])
            spans.append((len(pix), k))
            pix.append(image)
            if k:
                pix.append(crops)
        allp = torch.cat(pix, 0).contiguous() if len(pix) > 1 else pix[0]
        long_all, short_all = self.project_both(allp)
        nl, ns = c.clip_tokens, self.NLAT
        out, img_i = [], 0
        for (ids, image, crops, il, ol) in items:
            k = 0 if crops is None else int(crops.shape[0])
            img_long, img_short = long_all[img_i * nl:(img_i + 1) * nl], short_all[img_i * ns:(img_i + 1) * ns]
            obj_long, obj_short = long_all[(img_i + 1) * nl:(img_i + 1 + k) * nl], short_all[(img_i + 1) * ns:(img_i + 1 + k) * ns]
            img_i += 1 + k
            out.append(self._splice(list(ids), img_long, img_short, obj_long, obj_short, il, ol))
        return out

    def option_losses_batch(self, items):
        """Option scoring for several questions: items = [(question_ids, options_ids, image, object_crops, images_long,
        objects_long)] -> [(losses fp32 [n_options] on host, argmin)].

        The reference prefills the question once and then runs ONE FORWARD PER OPTION on its past_key_values
        (vstar_bench_eval.py:140-152).  Here every option of a question is scored in ONE pass: the options' tokens are
        appended back to back after the question's cache rows, every row carries its own RoPE position (Tq + index inside its
        option) and the attention masks the other options' rows (vsb_flash_attn_seg_bf16), so each row sees exactly the keys
        it sees in the reference.  Questions whose spliced length is equal are batched: one prefill with M = G*Tq rows and
        one option pass for all of them (each weight byte is read twice per GROUP instead of five times per question)."""
        embeds = self.build_embeds_batch([(q, img, crops, il, ol) for q, opts, img, crops, il, ol in items])
        groups = {}
        for i, x in enumerate(embeds):
            groups.setdefault(int(x.shape[0]), []).append(i)
        results = [None] * len(items)
        dev = self.dev
        for Tq, members in groups.items():
            G = len(members)
            opts = [[list(o) for o in items[i][1]] for i in members]
            Tn = max(sum(len(o) for o in oo) for oo in opts)
            self._ensure_cache(G, self._capacity(Tq + Tn))
            self._prefix_slots = 0
            x = torch.cat([embeds[i] for i in members], 0).contiguous() if G > 1 else embeds[members[0]]
            self._llm_layers(x, G, Tq, 0)
            self.kv_epoch = getattr(self, "kv_epoch", 0) + 1
            last = torch.tensor([g * Tq + Tq - 1 for g in range(G)], dtype=torch.int64, device=dev)
            _, _, q_last = self._logits_rows(x, last)                          # [G, V]: predicts the first token of every option
            # appended rows: options back to back, right-padded to Tn with rows that see only themselves
            ids = torch.zeros((G, Tn), dtype=torch.int64)
            pos = torch.zeros((G, Tn), dtype=torch.int32)
            seg = torch.zeros((G, Tn), dtype=torch.int32)
            pred, labels, spans = [], [], []
            for g, oo in enumerate(opts):
                off = 0
                for o in oo:
                    spans.append((g, len(labels), len(o)))
                    for j, tok in enumerate(o):
                        ids[g, off + j], pos[g, off + j], seg[g, off + j] = tok, Tq + j, Tq + off
                        pred.append(g if j == 0 else G + g * Tn + off + j - 1)
                        labels.append(tok)
                    off += len(o)
                for r in range(off, Tn):
                    pos[g, r], seg[g, r] = Tq, Tq + r
            xo = ops.gather_rows(ids.view(-1).to(dev), self.w.embed)
            self._llm_layers(xo, G, Tn, Tq, positions=pos.view(-1).to(dev), q_seg=seg.view(-1).to(dev), seg_lo=Tq)
            hn = ops.rmsnorm(xo, self.w.final_norm, self.cfg.rms_eps)
            lo = ops.gemm(hn, self.w.lm_head, out_dtype=torch.float32)
            rows = torch.cat([q_last, lo], 0).index_select(0, torch.tensor(pred, dtype=torch.int64, device=dev)).contiguous()
            nll = ops.nll_rows(rows, torch.tensor(labels, dtype=torch.int64, device=dev)).cpu()
            per = {}
            for g, s0, n in spans:
                per.setdefault(g, []).append(nll[s0:s0 + n].mean())
            for g, i in enumerate(members):
                losses = torch.stack(per[g])
                results[i] = (losses, int(losses.argmin()))
        return results


class StreamRequest:
    """handle of a request admitted to a DecodeStream: `tokens` grows by one id per step, `done` once it ended.
    A beam request (num_beams = k > 1) holds k cache `slots` (`slot` is the first); `beams` are its running beams' new ids while
    it decodes, and once it is done `tokens` / `score` are its chosen hypothesis' ids (eos appended as beam_search returns them)
    and score."""

    def __init__(self, rid, slot, length, max_new_tokens, stop_ids, temperature=0, top_k=0, top_p=None, seed=None, beam=None,
                 slots=None):
        self.id, self.slot, self.prompt_len = rid, slot, length
        self.max_new_tokens, self.stop_ids = max_new_tokens, list(stop_ids) if stop_ids else None
        self.tokens, self.done = [], False
        self.temperature, self.top_k, self.top_p, self.seed = temperature, top_k, top_p, seed     # temperature > 0: sampled
        self.beam = beam                                 # BeamRequest of a beam request
        self.slots = [slot] if slots is None else list(slots)
        self.beam_slot = [slot]                          # cache slot of each running beam, in beam order
        self.score = None
        self.preemptions = 0                             # times a growing paged stream swapped it out
        self.prefilled = length                          # prompt rows written to the cache (a chunked-prefill stream: 0 at admission)

    @property
    def prefilling(self):
        return self.prefilled < self.prompt_len

    @property
    def kind(self):
        return "beam" if self.beam is not None else "sample" if self.temperature > 0 else "greedy"

    @property
    def beams(self):
        return None if self.beam is None else [list(b) for b in self.beam.beams]

    def __repr__(self):
        return f"StreamRequest(id={self.id}, slot={self.slot}, kind={self.kind}, tokens={len(self.tokens)}, done={self.done})"


def _signed64(seed):
    """any integer seed -> the int64 with the same low 64 bits (the sampler's seed argument)"""
    return (int(seed) + (1 << 63)) % (1 << 64) - (1 << 63)


class DecodeStream:
    """Decoding of many requests on a decode batch that admits a new request whenever a slot frees (iteration-level
    admission), instead of generate_batch's static batch that steps until its longest answer ends.

    The stream owns its KV cache [n_layers, max_slots, max_positions, 3d], separate from the engine's, so option scoring,
    generate() or a VSM call in between neither disturbs it nor is disturbed by it.  A request is prefilled alone into a free
    slot at rows [0, T) and takes its first token from the prefill logits, as in generate().  Every step() then runs ONE
    vsb_llama_layers_slots call for all active rows (each row writes its new q|k|v at its own slot and length and attends
    only its own keys) and selects every row's next token into one device buffer, read by one device-to-host copy.  A request
    ends at eos, at its stop_ids (the rule of generate_batch) or after its own max_new_tokens, and its slot is free for the
    next admit().  In batch-invariant mode (ops.batch_invariant) a request's logits do not depend on the other requests in the
    batch or on its slot.

    Each request brings its own generation settings (admit): greedy (argmax_rows), sampled (temperature > 0: one
    vsb_sample_rows_var_f32 launch for every sampled row, each with its own temperature / top_k / top_p / seed / step) or beam
    search (num_beams = k: the request holds k slots; one vsb_beam_candidates_f32 launch per distinct k, and the forked beams'
    generated rows move by one vsb_copy_slot_rows_b16 launch).  Rows are ordered greedy, sampled, beam, each kind in slot
    order, so a greedy-only stream issues the launches it always did.

    kv_pages = N (paged mode): the cache is a pool [n_layers, N, PAGE_ROWS, 2d] of k|v pages instead of [max_slots,
    max_positions] rows per slot.  A slot is then a row of the device page table [max_slots, ceil(max_positions / PAGE_ROWS)]:
    max_slots bounds the rows decoded per step, max_positions one request, and a request reserves ceil((T + max_new_tokens) /
    PAGE_ROWS) pages at admission (a beam request shares its full prompt pages among its beams; kv_pages.PagePool).  A request
    is prefilled into a staging cache of its T rows and its k|v rows are written into its pages by one
    vsb_copy_page_rows_b16 launch; steps run vsb_llama_layers_slots_paged.  Logits and tokens are bit-identical to the
    contiguous stream's on the same admission schedule.  The page table is uploaded at admission, the only time it changes
    where a kernel could read it; a step still makes one device-to-host copy.

    kv_swap_pages = M (with kv_pages; growing mode): the stream also holds a swap area [M, n_layers, PAGE_ROWS, 2d] of pinned
    host memory, and a request takes only the pages its prompt fills at admission and one page per row whenever a step is about
    to write a page's first row (kv_pages.GrowingPool, which also states the admission rule).  When the free pages cannot
    cover a step's growth, the newest running request is preempted: vsb_swap_pages_b16 copies its pages to the swap area and
    they are free.  Preempted requests resume oldest first, before any new admission, on whichever pages and slots are free
    (their handles' `slot`, `slots` and beam slots change).  Swap copies run on the stream's CUDA stream in order with the
    steps; a step that changes the page table sends it in the step's one host-to-device upload.  Swapping keeps every bit, so
    in batch-invariant mode a request's logits do not depend on being preempted.  `preemptions`, `swapped_pages` (copied
    out) and `restored_pages` (copied back) count the traffic.

    prefill_chunk = C (with kv_pages, not with kv_swap_pages; chunked prefill): admit() reserves the request's pages and builds
    its embedding but runs no layer: the request is *prefilling* (handle.prefilled counts its prompt rows written, its
    `tokens` are empty).  Each step takes up to C prompt rows of the prefilling requests, first come first served
    (kv_pages.plan_chunks), and runs them after the running requests' decode rows in ONE vsb_llama_layers_chunked_paged call,
    so the running requests gain a token in every step while prompts are admitted.  A request whose last prompt row ran takes
    its first token from that row's logits in the same step, as admission gives it in the unchunked stream (argmax; (seed,
    step 0); a beam request copies its prompt rows from the last shared page on into its other beams' pages and selects its
    first candidates from k_in = 1).  lm_head runs on the decode rows and those last rows only.  In batch-invariant mode
    every token and logit equals the unchunked paged stream's on the same admission schedule for prompts of 64 rows or more
    (shorter prompts are prefilled there by the mma.sync attention kernel, which rounds differently)."""

    pages = None                                         # PagePool of a paged stream
    _swap = None                                         # pinned host swap area of a growing stream

    def __init__(self, engine, max_slots, max_positions, eos_token_id=2, kv_pages=None, kv_swap_pages=None, prefill_chunk=None):
        max_slots, max_positions = int(max_slots), int(max_positions)
        if max_slots < 1:
            raise ValueError(f"max_slots must be >= 1, got {max_slots}")
        if not 1 <= max_positions <= engine.MAX_POSITIONS:
            raise ops._lib.VsbError(f"max_positions {max_positions} outside [1, {engine.MAX_POSITIONS}] (the rows of the RoPE tables)")
        if kv_swap_pages is not None and kv_pages is None:
            raise ValueError("kv_swap_pages needs kv_pages: only a paged stream can swap its pages")
        if prefill_chunk is not None:
            if isinstance(prefill_chunk, bool) or int(prefill_chunk) != prefill_chunk or prefill_chunk < 1:
                raise ValueError(f"prefill_chunk must be an integer >= 1, got {prefill_chunk!r}")
            if kv_pages is None:
                raise ValueError("prefill_chunk needs kv_pages: prompt chunks are written through the page table")
            if kv_swap_pages is not None:
                raise ValueError("prefill_chunk does not combine with kv_swap_pages (a growing pool)")
            prefill_chunk = int(prefill_chunk)
        self.chunk = prefill_chunk
        self._prefilling = []                            # handles of the requests still prefilling, in admission order
        c = engine.cfg
        self.engine, self.eos = engine, eos_token_id
        self.max_slots, self.max_positions = max_slots, max_positions
        if engine._layer_table is None:
            engine._layer_table = ops.llama_layer_table(engine.w.layers)
        dev, dt = engine.dev, engine.dtype
        if kv_pages is None:
            self._cache = torch.empty((c.n_layers, max_slots, max_positions, 3 * c.hidden), dtype=dt, device=dev)
        elif kv_swap_pages is None:
            self.pages = PagePool(int(kv_pages), max_slots, pages_for(max_positions))
        else:
            self.pages = GrowingPool(int(kv_pages), max_slots, pages_for(max_positions), int(kv_swap_pages))
            self._swap = torch.empty((self.pages.swap_pages, c.n_layers, PAGE_ROWS, 2 * c.hidden), dtype=dt, pin_memory=True)
        if kv_pages is not None:
            self._cache = torch.empty((c.n_layers, self.pages.n_pages, PAGE_ROWS, 2 * c.hidden), dtype=dt, device=dev)
            self._page_table = torch.zeros(self.pages.table.shape, dtype=torch.int32, device=dev)
        rows = max_slots + (prefill_chunk or 0)          # a chunked step's decode rows plus at most C prompt rows
        self._scratch = torch.empty((rows * (5 * c.hidden + c.intermediate),), dtype=dt, device=dev)
        self._deq = torch.empty((2 * c.intermediate * c.hidden,), dtype=dt, device=dev) if getattr(engine.w, "quant", None) else None
        self._slots = [None] * max_slots                 # slot -> active StreamRequest (a beam request in each of its slots)
        self._finished = []                              # ended at admission; reported by the next step()
        self._next_id = 0
        self.steps = 0
        self.occupied = 0                                # sum over steps of the rows decoded
        self.last_logits = None                          # (requests in row order, fp32 logits [rows, V]) of the latest call
        self.preemptions = self.swapped_pages = self.restored_pages = 0
        self._preempted = {}                             # id -> handle of a request swapped out

    @property
    def growing(self):
        return isinstance(self.pages, GrowingPool)

    @property
    def free_slots(self):
        return sum(r is None for r in self._slots)

    def free_rows(self, k):
        """the first k free slots, or None when fewer are free"""
        rows = [i for i, r in enumerate(self._slots) if r is None]
        return rows[:k] if len(rows) >= k else None

    @property
    def active(self):
        """the running requests, in order of their first slot"""
        out, seen = [], set()
        for r in self._slots:
            if r is not None and r.id not in seen:
                seen.add(r.id)
                out.append(r)
        return out

    def _check_open(self):
        if self._cache is None:
            raise RuntimeError("decode stream is closed")

    def _ended(self, r):
        t = r.tokens
        return t[-1] == self.eos or (r.stop_ids and t[-len(r.stop_ids):] == r.stop_ids) or len(t) >= r.max_new_tokens

    def _release(self, r):
        r.done = True
        for s in r.slots:
            self._slots[s] = None
        if self.growing:
            self.pages.finish(r.id)
        elif self.pages is not None:
            self.pages.release(r.slots)

    def _beam_advance(self, r, cand):
        """one beam-search step of request r on its 2k candidates [(score, token, beam)] -> the (src, dst, lo, hi) row copies of
        its forks, or None when it ended (tokens / score then hold its chosen hypothesis)"""
        q = r.beam
        n = len(q.beams[0])                              # tokens every beam had before this step: rows [T, T + n) are cached
        nxt = q.process(cand)
        r.beam_slot, forks = fork_slots(r.beam_slot, nxt, r.slots)
        if q.done or len(q.beams[0]) >= r.max_new_tokens:
            r.tokens, r.score = q.finalize()
            return None
        return [(a, b, r.prompt_len, r.prompt_len + n) for a, b in forks] if n else []

    def admit(self, request, max_new_tokens, stop_ids=None, *, temperature=0, top_k=DEFAULT_TOP_K, top_p=None, seed=None, num_beams=1,
              length_penalty=DEFAULT_LENGTH_PENALTY, early_stopping=DEFAULT_EARLY_STOPPING):
        """request = (input_ids, image, object_crops, images_long, objects_long) as generate_batch takes it -> StreamRequest.
        The settings are generate()'s for this request alone: greedy by default; temperature > 0 samples with top_k / top_p
        (check_sampling), token t drawn with (seed, step t), seed None = one draw from torch's default generator;
        num_beams = k > 1 runs beam_search's scorer with length_penalty / early_stopping on k slots (stop_ids at most [eos]),
        its first candidates selected here from the prefill logits.  Raises (before any launch) on settings generate() refuses,
        when fewer than num_beams slots are free, num_beams exceeds max_slots or the prompt plus max_new_tokens exceeds
        max_positions, and in paged mode when the free pages are fewer than the request reserves (RuntimeError; in growing
        mode also while preempted requests wait and when kv_pages.GrowingPool's admission rule refuses)."""
        self._check_open()
        ids, image, crops, il, ol = request
        max_new_tokens = int(max_new_tokens)
        if max_new_tokens < 1:
            raise ValueError(f"max_new_tokens must be >= 1, got {max_new_tokens}")
        e = self.engine
        beam = e._beam_args(num_beams, temperature, stop_ids, self.eos, early_stopping)
        sample = not beam and temperature is not None and temperature > 0
        if sample:
            top_k, top_p = check_sampling(top_k, top_p)
        k = num_beams
        if k > self.max_slots:
            raise ValueError(f"num_beams = {k} needs {k} slots, the decode stream has {self.max_slots}")
        T = e.spliced_length(ids, 0 if crops is None else int(crops.shape[0]), il, ol)
        if T + max_new_tokens > self.max_positions:
            raise ops._lib.VsbError(f"prompt of {T} rows + {max_new_tokens} new tokens exceeds the stream's {self.max_positions} "
                                    "positions per slot")
        if self.free_slots < k:
            raise RuntimeError(f"no free slot: all {self.max_slots} slots of the decode stream are in use" if k == 1 else
                               f"no free slot for {k} beams: {self.free_slots} of the decode stream's {self.max_slots} slots are free")
        slots = [i for i, r in enumerate(self._slots) if r is None][:k]
        if self.growing:
            self.pages.check_admit(slots, T, max_new_tokens)
        elif self.pages is not None:
            self.pages.check_reserve(slots, T, max_new_tokens)
        if sample and seed is None:
            seed = draw_seeds(1)[0]
        slot = slots[0]
        x = e.build_embeds(ids, image, crops, il, ol)
        assert x.shape[0] == T
        if self.chunk is not None:
            return self._admit_chunked(x, T, max_new_tokens, stop_ids, slots, sample, temperature, top_k, top_p, seed, beam, k, len(ids),
                                       length_penalty, early_stopping)
        c = e.cfg
        scratch = torch.empty((T * (2 * c.hidden + c.intermediate),), dtype=e.dtype, device=e.dev)
        if self.pages is None:
            Bc, Tm = self.max_slots, self.max_positions
            ops.llama_layers(e._layer_table, len(e.w.layers), x, 1, T, 0, self._cache, Bc, Tm, c.hidden, c.n_heads, c.intermediate,
                             c.rms_eps, e.w.rope_cos, e.w.rope_sin, scratch, cache_row_offset=slot * Tm,
                             norm_folded=getattr(e.w, "fold_norms", False), deq_scratch=self._deq)
        else:
            self._admit_paged(x, T, max_new_tokens, slots, scratch)
        _, idx, logits = e._logits_rows(x, torch.tensor([T - 1], dtype=torch.int64, device=e.dev))
        r = StreamRequest(self._next_id, slot, T, max_new_tokens, stop_ids, temperature=float(temperature) if sample else 0,
                          top_k=top_k if sample else 0, top_p=top_p if sample else None, seed=seed if sample else None,
                          beam=BeamRequest(k, len(ids), max_new_tokens, self.eos, length_penalty, early_stopping) if beam else None,
                          slots=slots)
        self._next_id += 1
        self.last_logits = ([r], logits)
        for s in slots:
            self._slots[s] = r
        if beam:
            if self.pages is None:
                ops.copy_slot_rows(self._cache, [(slot, s, 0, T) for s in slots[1:]])      # the prompt rows of the other beams
            dev = e.dev
            cand = ops.beam_candidates(logits, torch.zeros((1, 1), dtype=torch.int32, device=dev),
                                       torch.zeros((1, 1), dtype=torch.float32, device=dev), k, e.dtype).cpu()
            ended = self._beam_advance(r, list(zip(cand[0, 0].view(torch.float32).tolist(), cand[1, 0].tolist(), cand[2, 0].tolist()))) is None
        else:
            if sample:
                sd = torch.tensor([_signed64(seed)], dtype=torch.int64, device=e.dev)
                idx = ops.sample_rows(logits, r.temperature, top_k, top_p, e.dtype, sd, 0)
            r.tokens.append(int(idx[0]))
            ended = self._ended(r)
        if ended:
            self._release(r)
            self._finished.append(r)
        return r

    def _admit_chunked(self, x, T, max_new_tokens, stop_ids, slots, sample, temperature, top_k, top_p, seed, beam, k, n_ids, length_penalty,
                       early_stopping):
        """a chunked-prefill stream's admission: the request's pages and its embedding x [T, d], held until step() has run its
        last prompt row"""
        shared = self.pages.reserve(slots, T, max_new_tokens)
        self._page_table.copy_(torch.from_numpy(self.pages.table))
        r = StreamRequest(self._next_id, slots[0], T, max_new_tokens, stop_ids, temperature=float(temperature) if sample else 0,
                          top_k=top_k if sample else 0, top_p=top_p if sample else None, seed=seed if sample else None,
                          beam=BeamRequest(k, n_ids, max_new_tokens, self.eos, length_penalty, early_stopping) if beam else None,
                          slots=slots)
        r.prefilled, r._x, r._shared = 0, x, shared
        self._next_id += 1
        for s in slots:
            self._slots[s] = r
        self._prefilling.append(r)
        return r

    def _admit_paged(self, x, T, max_new_tokens, slots, scratch):
        """prefill x [T, d] into a staging cache of T rows with the contiguous runner, reserve the request's pages and write
        its k|v rows into them: all T rows into the first beam's pages (the shared full pages among them), rows from the
        last shared page on into every other beam's private pages"""
        e, c = self.engine, self.engine.cfg
        staging = torch.empty((c.n_layers, 1, T, 3 * c.hidden), dtype=e.dtype, device=e.dev)
        ops.llama_layers(e._layer_table, len(e.w.layers), x, 1, T, 0, staging, 1, T, c.hidden, c.n_heads, c.intermediate, c.rms_eps,
                         e.w.rope_cos, e.w.rope_sin, scratch, norm_folded=getattr(e.w, "fold_norms", False), deq_scratch=self._deq)
        if self.growing:
            shared = self.pages.admit(self._next_id, slots, T, max_new_tokens)
        else:
            shared = self.pages.reserve(slots, T, max_new_tokens)
        self._page_table.copy_(torch.from_numpy(self.pages.table))
        lo = shared * PAGE_ROWS
        ops.copy_page_rows(self._cache, self._page_table, [(0, slots[0], 0, T)] + [(0, s, lo, T) for s in slots[1:]],
                           src=staging[..., c.hidden:])

    def step(self):
        """one decode step of every active request -> [(handle, new token ids)] of the requests that ended in it (and of those
        that ended at admission since the previous step)"""
        self._check_open()
        done, self._finished = [(r, r.tokens) for r in self._finished], []
        table = self._schedule() if self.growing else False
        act = self.active
        if not act:
            return done
        e, c = self.engine, self.engine.cfg
        if self.chunk is not None:
            act = [r for r in act if not r.prefilling]
            segs = plan_chunks([(r, r.prefilled, r.prompt_len) for r in self._prefilling], self.chunk)
        else:
            segs = []
        comp = [r for r, lo, n in segs if lo + n == r.prompt_len]     # prompts complete in this step: their first token is due
        greedy = [r for r in act if r.kind == "greedy"]
        sampled = [r for r in act if r.kind == "sample"]
        beams = [r for r in act if r.kind == "beam"]
        # rows (request, slot, rows cached, newest token): the newest token goes to row `rows cached` of the slot
        rows = [(r, r.slot, r.prompt_len + len(r.tokens) - 1, r.tokens[-1]) for r in greedy + sampled]
        first = {}                                       # beam request -> its first logits row
        for r in beams:
            first[r.id] = len(rows)
            n = r.prompt_len + len(r.beam.beams[0]) - 1
            rows += [(r, s, n, b[-1]) for s, b in zip(r.beam_slot, r.beam.beams)]
        B = len(rows)
        lens = [n for _, _, n, _ in rows]
        if segs:
            return self._step_chunked(done, rows, greedy, sampled, beams, first, segs, comp)
        meta = np.array([[s for _, s, _, _ in rows], lens, lens], dtype=np.int32)
        if table:                                        # the grown page table travels with the step's metadata
            up = torch.from_numpy(np.concatenate([meta.ravel(), self.pages.table.ravel()])).to(e.dev)
            meta, self._page_table = up[:3 * B].view(3, B), up[3 * B:].view(self.pages.table.shape)
        else:
            meta = torch.from_numpy(meta).to(e.dev)
        ids = torch.tensor([t for _, _, _, t in rows], dtype=torch.int64).to(e.dev)
        x = ops.gather_rows(ids, e.w.embed)
        if self.pages is None:
            ops.llama_layers_slots(e._layer_table, len(e.w.layers), x, self._cache, c.rms_eps, e.w.rope_cos, e.w.rope_sin, self._scratch,
                                   meta[0], meta[1], meta[2], max(lens), c.n_heads, c.intermediate,
                                   norm_folded=getattr(e.w, "fold_norms", False), deq_scratch=self._deq)
        else:
            ops.llama_layers_slots_paged(e._layer_table, len(e.w.layers), x, self._cache, self._page_table, c.rms_eps, e.w.rope_cos,
                                         e.w.rope_sin, self._scratch, meta[0], meta[1], meta[2], max(lens), c.n_heads, c.intermediate,
                                         norm_folded=getattr(e.w, "fold_norms", False), deq_scratch=self._deq)
        hn = ops.rmsnorm(x, e.w.final_norm, c.rms_eps)
        logits = ops.gemm(hn, e.w.lm_head, out_dtype=torch.float32)
        groups = {}                                      # (k, beams in) -> beam requests of that k, in row order
        for r in beams:
            groups.setdefault((r.beam.k, r.beam.k), []).append(r)
        return self._finish_step(done, logits, greedy, sampled, groups, first, [r for r, _, _, _ in rows], B)

    def _step_chunked(self, done, rows, greedy, sampled, beams, first, segs, comp):
        """step() of a chunked-prefill stream whose step carries prompt rows (segs: kv_pages.plan_chunks' segments; comp: the
        requests whose prompt completes)"""
        e, c = self.engine, self.engine.cfg
        B, R, S = len(rows), sum(n for _, _, n in segs), len(segs)
        # logits rows: greedy decode rows then the greedy prompts completing, the same for sampled, then the beam decode rows and
        # each completing beam request's one row (its first candidates are taken from k_in = 1); gather picks them from x
        end, o = {}, B
        for r, lo, n in segs:
            o += n
            end[r.id] = o - 1
        cg, cs, cb = ([r for r in comp if r.kind == kd] for kd in ("greedy", "sample", "beam"))
        G0, S0 = len(greedy), len(sampled)
        pick = list(range(G0)) + [end[r.id] for r in cg] + list(range(G0, G0 + S0)) + [end[r.id] for r in cs] + \
            list(range(G0 + S0, B)) + [end[r.id] for r in cb]
        nb = len(pick) - B                                # logits rows past the decode rows' own
        shift = {r.id: first[r.id] + len(cg) + len(cs) for r in beams}
        for i, r in enumerate(cb):
            shift[r.id] = len(pick) - len(cb) + i
        lens = [n for _, _, n, _ in rows] + [lo + i for r, lo, n in segs for i in range(n)]
        slots = [s for _, s, _, _ in rows] + [r.slot for r, lo, n in segs for _ in range(n)]
        # one upload: the gather rows (int64, first so their view is aligned), slot / len / pos of every row, the segments
        host = np.empty(2 * len(pick) * (nb > 0) + 3 * (B + R) + 3 * S, dtype=np.int32)
        q = 2 * len(pick) * (nb > 0)
        if nb:
            host[:q].view(np.int64)[:] = pick
        host[q:q + 3 * (B + R)] = np.array([slots, lens, lens], dtype=np.int32).ravel()
        host[q + 3 * (B + R):] = np.array([[r.slot for r, _, _ in segs], [lo for _, lo, _ in segs], [n for _, _, n in segs]],
                                          dtype=np.int32).ravel()
        up = torch.from_numpy(host).to(e.dev)
        meta = up[q:q + 3 * (B + R)].view(3, B + R)
        seg = up[q + 3 * (B + R):].view(3, S)
        x = torch.empty((B + R, c.hidden), dtype=e.dtype, device=e.dev)
        if B:
            ids = torch.tensor([t for _, _, _, t in rows], dtype=torch.int64).to(e.dev)
            ops.gather_rows(ids, e.w.embed, out=x[:B])
        o = B
        for r, lo, n in segs:
            ops.copy2d(r._x[lo:lo + n], x[o:o + n])
            o += n
        ops.llama_layers_chunked_paged(e._layer_table, len(e.w.layers), x, self._cache, self._page_table, c.rms_eps, e.w.rope_cos,
                                       e.w.rope_sin, self._scratch, meta[0], meta[1], meta[2], max(lens[:B], default=0), seg, R,
                                       c.n_heads, c.intermediate, norm_folded=getattr(e.w, "fold_norms", False), deq_scratch=self._deq)
        for r, lo, n in segs:
            r.prefilled = lo + n
        for r in comp:
            self._prefilling.remove(r)
            r._x = None
            if r.kind == "beam" and len(r.slots) > 1:   # the prompt rows from the last shared page on, into the other beams' pages
                ops.copy_page_rows(self._cache, self._page_table, [(r.slots[0], s, r._shared * PAGE_ROWS, r.prompt_len) for s in r.slots[1:]])
        if not pick:
            self.steps += 1
            self.last_logits = None
            return done
        hn = ops.rmsnorm(ops.gather_rows(up[:q].view(torch.int64), x) if nb else x[:B], e.w.final_norm, c.rms_eps)
        logits = ops.gemm(hn, e.w.lm_head, out_dtype=torch.float32)
        groups = {}
        for r in beams:
            groups.setdefault((r.beam.k, r.beam.k), []).append(r)
        for r in cb:
            groups.setdefault((r.beam.k, 1), []).append(r)
        order = [r for r, _, _, _ in rows[:G0]] + cg + [r for r, _, _, _ in rows[G0:G0 + S0]] + cs + [r for r, _, _, _ in rows[G0 + S0:]] + cb
        return self._finish_step(done, logits, greedy + cg, sampled + cs, groups, shift, order, B)

    def _finish_step(self, done, logits, greedy, sampled, groups, first, order, B):
        """the selections of a step's logits rows (greedy rows, then sampled ones, then every beam group's rows), its one
        device-to-host copy, and the requests' advance -> done"""
        e = self.engine
        G, S = len(greedy), len(sampled)
        sel = torch.empty((G + S + sum(3 * len(g) * 2 * k for (k, _), g in groups.items()),), dtype=torch.int32, device=e.dev)
        if G:
            ops.argmax_rows(logits[:G], out=sel[:G])
        if S or groups:
            self._select(logits, G, sampled, groups, first, sel)
        h = sel.cpu()                                    # the one device-to-host copy of the step
        self.last_logits = (order, logits)
        self.steps += 1
        self.occupied += B
        for r, t in zip(greedy + sampled, h[:G + S].tolist()):
            r.tokens.append(int(t))
            if self._ended(r):
                self._release(r)
                done.append((r, r.tokens))
        off, quads = G + S, []
        for (k, _), g in groups.items():
            R = len(g)
            cand = h[off:off + 3 * R * 2 * k].view(3, R, 2 * k)
            off += 3 * R * 2 * k
            sc, tok, bm = cand[0].view(torch.float32).tolist(), cand[1].tolist(), cand[2].tolist()
            for i, r in enumerate(g):
                q = self._beam_advance(r, list(zip(sc[i], tok[i], bm[i])))
                if q is None:
                    self._release(r)
                    done.append((r, r.tokens))
                else:
                    quads += q
        for i in range(0, len(quads), ops.COPY_ROWS_MAX_PAIRS):
            if self.pages is None:
                ops.copy_slot_rows(self._cache, quads[i:i + ops.COPY_ROWS_MAX_PAIRS])
            else:
                ops.copy_page_rows(self._cache, self._page_table, quads[i:i + ops.COPY_ROWS_MAX_PAIRS])
        return done

    def _select(self, logits, G, sampled, groups, first, sel):
        """the sampled and beam rows' selections into sel[G:] (after the greedy rows' tokens): one per-row sampler launch for
        rows [G, G + S), then one candidate launch per beam width k (first: each beam request's first logits row); their
        settings travel in one host-to-device copy"""
        e, S = self.engine, len(sampled)
        nb = sum(len(g) * kin for (k, kin), g in groups.items())
        host = np.empty(6 * S + 2 * nb, dtype=np.int32)                       # seeds (int64) first, so their view is aligned
        host[:2 * S].view(np.int64)[:] = [_signed64(r.seed) for r in sampled]
        host[2 * S:3 * S].view(np.float32)[:] = [r.temperature for r in sampled]
        host[3 * S:4 * S] = [r.top_k for r in sampled]
        host[4 * S:5 * S].view(np.float32)[:] = [1.0 if r.top_p is None else r.top_p for r in sampled]
        host[5 * S:6 * S] = [len(r.tokens) for r in sampled]                  # token t is drawn at step t
        o, spans = 6 * S, []
        for (k, kin), g in groups.items():
            n = len(g) * kin
            host[o:o + n] = [first[r.id] + b for r in g for b in range(kin)]   # each request's beams, in beam order
            # kin = 1: a prompt completed in this step, its first candidates from one row of score 0
            host[o + n:o + 2 * n].view(np.float32)[:] = [s for r in g for s in (r.beam.scores if kin == k else [0.0])]
            spans.append((k, len(g), o, n))
            o += 2 * n
        dev = torch.from_numpy(host).to(e.dev)
        if S:
            ops.sample_rows_var(logits[G:G + S], dev[2 * S:3 * S].view(torch.float32), dev[3 * S:4 * S],
                                dev[4 * S:5 * S].view(torch.float32), e.dtype, dev[:2 * S].view(torch.int64), dev[5 * S:6 * S],
                                out=sel[G:G + S])
        off = G + S
        for k, R, o, n in spans:
            ops.beam_candidates(logits, dev[o:o + n].view(R, n // R), dev[o + n:o + 2 * n].view(torch.float32).view(R, n // R), k, e.dtype,
                                out=sel[off:off + 3 * R * 2 * k].view(3, R, 2 * k))
            off += 3 * R * 2 * k

    def _schedule(self):
        """a growing stream's page work before a step (GrowingPool.schedule): swap preempted requests back in or the newest
        running ones out, then grow -> whether the page table changed"""
        running = {r.id: r for r in self._slots if r is not None}
        resumed, preempted, changed = self.pages.schedule()
        for key, pairs in preempted:
            r = running[key]
            ops.swap_pages(self._cache, self._swap, pairs, to_host=True)
            for s in r.slots:
                self._slots[s] = None
            r.preemptions += 1
            self.preemptions += 1
            self.swapped_pages += len(pairs)
            self._preempted[key] = r
        for key, rows, pairs in resumed:
            r = self._preempted.pop(key)
            ops.swap_pages(self._cache, self._swap, [(p, s) for s, p in pairs], to_host=False)
            new = dict(zip(r.slots, rows))
            r.slots, r.slot, r.beam_slot = list(rows), rows[0], [new[s] for s in r.beam_slot]
            for s in rows:
                self._slots[s] = r
            self.restored_pages += len(pairs)
        return changed

    def close(self):
        """free the stream's cache and scratch (requests still running are abandoned; in paged mode their pages return to the
        pool, and a growing stream's swap area is freed)"""
        self._cache = self._scratch = self._deq = self._page_table = self._swap = None
        self._preempted = {}
        self._prefilling = []
        if self.pages is not None:
            self.pages.release_all()
        self._slots = [None] * self.max_slots
        self.last_logits = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


# ----------------------------------------------------------------------------------------------------------------
def _clip_preprocess(pil_img, size=224):
    """CLIPImageProcessor.preprocess of the reference (shortest edge 224 bicubic, centre crop 224, /255, mean/std)"""
    from PIL import Image
    img = pil_img.convert("RGB")
    w, h = img.size
    short = min(w, h)
    if (w, h) != (size, size):
        nw, nh = int(w * size / short), int(h * size / short)
        img = img.resize((nw, nh), resample=Image.BICUBIC)
        left, top = (nw - size) // 2, (nh - size) // 2
        img = img.crop((left, top, left + size, top + size))
    out = torch.empty((3, size, size), dtype=torch.float32)
    _normalize_into(np.array(img), out)
    return out


class _Proc:
    crop_size = {"height": 224, "width": 224}
    image_mean = list(CLIP_MEAN)

    def preprocess(self, image, return_tensors="pt"):
        return {"pixel_values": [_clip_preprocess(image)]}


class _ModelConfig:
    pass


class _ModelOutput:
    def __init__(self, logits, past_key_values):
        self.logits, self.past_key_values = logits, past_key_values


class _Past:
    """opaque `past_key_values`: the KV rows live in the engine's cache; this records how many are valid and which prefill
    wrote them (a handle from before a later prefill is rejected instead of silently reading the wrong rows)"""

    def __init__(self, length, epoch):
        self.length, self.epoch = length, epoch


class LlavaSearchModel:
    """The `model` that load_pretrained_model returns: the part of LlavaSearchLlamaForCausalLM's surface that
    /root/reference/vstar_bench_eval.py drives (generate(...) at :91-103; forward with images / with past_key_values at
    :127-152; .config.vocab_size at :157), on the sm_90a engine.  Greedy decoding only (the benchmark uses temperature 0)."""

    def __init__(self, engine: VQAEngine, eos_token_id=2):
        self.engine = engine
        self.config = _ModelConfig()
        self.config.vocab_size = engine.cfg.vocab
        self.eos_token_id = eos_token_id
        self.device = torch.device(engine.dev)
        self.top_k = DEFAULT_TOP_K                      # the top_k VQA_LLM samples with (generation_config.json's, if any)
        self.length_penalty = DEFAULT_LENGTH_PENALTY    # beam-search settings (generation_config.json's, if any)
        self.early_stopping = DEFAULT_EARLY_STOPPING

    def eval(self):
        return self

    def cuda(self):
        return self

    def _px(self, t):
        if t is None or len(t) == 0:
            return None
        return ops.cast_f32(torch.as_tensor(t).float().to(self.engine.dev).contiguous(), self.engine.dtype)

    @torch.inference_mode()
    def generate(self, input_ids, images=None, object_features=None, images_long=None, objects_long=None, do_sample=False, num_beams=1,
                 temperature=0, top_p=None, max_new_tokens=200, use_cache=True, stopping_criteria=None, length_penalty=None,
                 early_stopping=None, **_):
        """greedy decoding, or beam search with num_beams > 1 (HF's output: prompt ids + the chosen hypothesis + eos when it is
        shorter than max_length; stopping_criteria see the k running beams as a [k, len] tensor in beam order, as HF's do).
        length_penalty / early_stopping None: the checkpoint's generation_config.json values (else the 4.31 defaults)."""
        if do_sample:
            raise NotImplementedError("greedy decoding only (vstar_bench_eval.py:196 runs temperature=0, num_beams=1)")
        check_beams(num_beams, self.early_stopping if early_stopping is None else early_stopping)
        ids = input_ids.view(-1).tolist()
        stop_fn = None
        if stopping_criteria:
            def stop_fn(new):
                new = [list(new)] if num_beams == 1 else new
                full = torch.tensor([ids + list(b) for b in new], dtype=torch.int64)
                return any(bool(sc(full, None)) for sc in stopping_criteria)
        beam = {} if num_beams == 1 else dict(
            num_beams=num_beams, length_penalty=self.length_penalty if length_penalty is None else length_penalty,
            early_stopping=self.early_stopping if early_stopping is None else early_stopping)
        new = self.engine.generate(ids, self._px(images), self._px(object_features), images_long, objects_long, max_new_tokens,
                                   self.eos_token_id, stop_fn=stop_fn, **beam)
        return torch.cat([input_ids.view(1, -1).cpu(), torch.tensor([new], dtype=torch.int64)], dim=1).to(input_ids.device)

    @torch.inference_mode()
    def __call__(self, input_ids=None, use_cache=True, images=None, object_features=None, images_long=None, objects_long=None,
                 attention_mask=None, past_key_values=None, **_):
        e = self.engine
        if past_key_values is None:
            x = e.build_embeds(input_ids.view(-1).tolist(), self._px(images), self._px(object_features), images_long, objects_long)
            T = x.shape[0]
            e.prefill_embeds(x)
            _, _, logits = e._logits_rows(x, torch.arange(T, dtype=torch.int64, device=e.dev))
            return _ModelOutput(logits.view(1, T, -1), _Past(T, e.kv_epoch))
        if past_key_values.epoch != e.kv_epoch:
            raise RuntimeError("stale past_key_values: the engine's KV cache has been re-prefilled since this handle was returned")
        toks = input_ids.view(-1).tolist()
        logits = e.append_tokens(toks, past_key_values.length)          # rows of an earlier continuation are overwritten
        return _ModelOutput(logits.view(1, len(toks), -1), _Past(past_key_values.length + len(toks), e.kv_epoch))


def load_pretrained_model(model_path, model_base=None, model_name=None, load_8bit=False, load_4bit=False, device_map="auto",
                          device="cuda", torch_dtype=None):
    """Drop-in for /root/reference/LLaVA/llava/model/builder.py:26-151 (the SEAL VQA LLM branch):
    -> (tokenizer, model, image_processor, context_len).  model_path: local `seal_vqa_7b` checkpoint directory (HF
    safetensors / .bin shards in the reference's key layout).
    torch_dtype: None / torch.bfloat16 (default) or torch.float16 (the reference's dtype, builder.py:43) for the engine.
    load_4bit: the reference's bitsandbytes NF4 mode (builder.py:33-40): every Llama and projector Linear in NF4 with
    double-quantised scales, CLIP / embeddings / lm_head / norms / biases in fp16, compute in fp16 (torch_dtype None or fp16).
    load_8bit (LLM.int8 with outlier decomposition) is not implemented."""
    import os
    if load_8bit:
        raise NotImplementedError("load_8bit (bitsandbytes LLM.int8) is not implemented; load_4bit (NF4) is")
    if load_4bit and torch_dtype not in (None, torch.float16):
        raise ValueError(f"load_4bit computes in fp16 (the reference's bnb_4bit_compute_dtype), got torch_dtype={torch_dtype}")
    if not os.path.isdir(str(model_path)):
        raise FileNotFoundError("load_pretrained_model: model_path must be a local checkpoint directory (no network here)")
    from transformers import AutoTokenizer
    from .vsm import config_from_hf, open_checkpoint
    tokenizer = AutoTokenizer.from_pretrained(model_path, use_fast=False)
    cfg = config_from_hf(model_path)
    dtype = torch.float16 if load_4bit else (BF if torch_dtype is None else torch_dtype)
    engine = VQAEngine(VQAWeights(cfg, open_checkpoint(model_path, device=device), device=device, dtype=dtype,
                                  quant="nf4" if load_4bit else None))
    model = LlavaSearchModel(engine, getattr(tokenizer, "eos_token_id", 2))
    model.top_k, model.length_penalty, model.early_stopping = generation_top_k(model_path, beams=True)
    return tokenizer, model, _Proc(), 2048


class VQA_LLM:
    """Same surface as /root/reference/vstar_bench_eval.py:38-165.  args.vqa_dtype (optional): "bf16" (default) or "fp16";
    args.vqa_load_4bit (optional): NF4 Linear weights, fp16 compute (load_pretrained_model(load_4bit=True))."""

    def __init__(self, args=None, engine: VQAEngine = None, tokenizer=None, conv_type="v1"):
        if engine is None:
            name = getattr(args, "vqa_dtype", None) or "bf16"
            if name not in VQA_DTYPES:
                raise ValueError(f"vqa_dtype must be one of {sorted(VQA_DTYPES)}, got {name!r}")
            load_4bit = bool(getattr(args, "vqa_load_4bit", False))      # NF4 computes in fp16 whatever vqa_dtype says
            self.tokenizer, self.model, self.image_processor, self.context_len = load_pretrained_model(
                args.vqa_model_path, None, None, load_4bit=load_4bit, torch_dtype=None if load_4bit else VQA_DTYPES[name])
            self.engine = self.model.engine
            self.top_k = self.model.top_k
            self.length_penalty, self.early_stopping = self.model.length_penalty, self.model.early_stopping
            self.conv_type = getattr(args, "conv_type", "v1")
            self.eos = getattr(self.tokenizer, "eos_token_id", 2)
            return
        self.engine = engine
        self.model = LlavaSearchModel(engine)
        self.tokenizer = tokenizer if tokenizer is not None else SyntheticTokenizer(engine.cfg)
        self.image_processor = _Proc()
        self.context_len = 2048
        self.top_k = DEFAULT_TOP_K
        self.length_penalty, self.early_stopping = DEFAULT_LENGTH_PENALTY, DEFAULT_EARLY_STOPPING
        self.conv_type = conv_type
        self.eos = getattr(self.tokenizer, "eos_token_id", 2)

    _img_src = None

    def get_patch(self, bbox, image_width, image_height, patch_size=224, patch_scale=None):
        object_width = int(np.ceil(bbox[2]))
        object_height = int(np.ceil(bbox[3]))
        cx = int(bbox[0] + bbox[2] / 2)
        cy = int(bbox[1] + bbox[3] / 2)
        if patch_scale is None:
            pw, ph = max(object_width, patch_size), max(object_height, patch_size)
        else:
            pw, ph = int(object_width * patch_scale), int(object_height * patch_scale)
        left = max(0, cx - pw // 2)
        right = min(left + pw, image_width)
        top = max(0, cy - ph // 2)
        bottom = min(top + ph, image_height)
        return [left, top, right, bottom]

    def get_object_crop(self, image, bbox, patch_scale):
        b = self.get_patch(bbox, image.width, image.height, patch_scale=patch_scale)
        crop = image.crop((b[0], b[1], b[2], b[3])).resize((224, 224))
        return _clip_preprocess(crop)

    def _pixels(self, image, object_crops):
        if torch.is_tensor(image) and image.is_cuda:            # already preprocessed on the device (device_pixels)
            return image, object_crops
        img = _clip_preprocess(image).unsqueeze(0).to(self.engine.dev)
        img = ops.cast_f32(img.contiguous(), self.engine.dtype)
        crops = None
        if object_crops is not None and len(object_crops) > 0:
            crops = ops.cast_f32(torch.as_tensor(object_crops).float().to(self.engine.dev).contiguous(), self.engine.dtype)
        return img, crops

    def use_device_images(self, vsm):
        """share the VSM's resident search images and its Pillow-exact GPU resize pipeline: the padded image and the object
        crops of the option-scoring prompt (vstar_bench_eval.py:228-256) are then cut and resized on the device from the
        image that is already in HBM - bit-identical pixels, no host PIL work between the search and the answer"""
        self._img_src = vsm

    def device_pixels(self, image, boxes, patch_scale=1.2):
        """== (_clip_preprocess(expand2square_center(image)), [get_object_crop(image, b, patch_scale) for b in boxes]) as device
        tensors of the engine dtype ([1,3,224,224], [k,3,224,224] or None), computed by the GPU image pipeline.  fp16: the
        pipeline's fp32 normalised pixels cast to fp16, i.e. the reference's .half() of its fp32 pixel tensor"""
        vsm = self._img_src
        pipe = vsm.pipeline
        res = vsm.resident(image)                                   # uint8 [H, W, 3] in HBM
        H, W = int(res.shape[0]), int(res.shape[1])
        side = max(W, H)
        dev = self.engine.dev
        f16 = self.engine.dtype == torch.float16

        def resize(src_, l, t, w, h, iw, ih, out):
            if f16:
                f32 = torch.empty(out.shape, dtype=torch.float32, device=dev)
                pipe._resize(src_, l, t, w, h, iw, ih, 224, 224, out_f32=f32)
                ops.cast_f32(f32, torch.float16, out=out)
            else:
                pipe._resize(src_, l, t, w, h, iw, ih, 224, 224, out_bf16=out)

        img = torch.empty((1, 3, 224, 224), dtype=self.engine.dtype, device=dev)
        if W == H:
            src = res
        else:                                                       # centred padding (vstar_bench_eval.py:25-36)
            bg = torch.tensor([int(x * 255) for x in self.image_processor.image_mean], dtype=torch.uint8, device=dev)
            src = bg.view(1, 1, 3).expand(side, side, 3).contiguous()
            left, top = (side - W) // 2, (side - H) // 2
            src[top:top + H, left:left + W] = res
        resize(src, 0, 0, side, side, side, side, img[0])
        crops = None
        if boxes is not None and len(boxes) > 0:
            crops = torch.empty((len(boxes), 3, 224, 224), dtype=self.engine.dtype, device=dev)
            for i, b in enumerate(boxes):
                l, t, r, btm = self.get_patch(b, W, H, patch_scale=patch_scale)
                resize(res, l, t, r - l, btm - t, r - l, btm - t, crops[i])
        return img, crops

    @torch.inference_mode()
    def free_form_inference(self, image, question, temperature=0, top_p=None, num_beams=1, max_new_tokens=200, object_crops=None,
                            images_long=None, objects_long=None):
        """temperature > 0 samples (the reference's do_sample = temperature > 0, vstar_bench_eval.py:97) with top_k = self.top_k
        and top_p; the request takes one seed from torch's default generator.  num_beams > 1: beam search with
        self.length_penalty / self.early_stopping; eos ends a hypothesis, and no other stopping criterion applies (the
        v1 stop keyword "</s>" is eos; the reference's KeywordsStoppingCriteria would assert on k beams, INTEGRATION.md)"""
        sample = temperature is not None and temperature > 0
        if sample:
            check_sampling(self.top_k, top_p)
        if num_beams != 1:
            return self._beam_texts([(image, question, object_crops, images_long, objects_long)], num_beams, max_new_tokens, temperature)[0]
        ids = self._prompt_ids(question)
        img, crops = self._pixels(image, object_crops)
        out = self.engine.generate(ids, img, crops, images_long, objects_long, max_new_tokens, self.eos, stop_ids=self._stop_ids(),
                                   temperature=temperature if sample else 0, top_k=self.top_k, top_p=top_p,
                                   seed=draw_seeds(1)[0] if sample else None)
        return self._answer_text(out)

    @torch.inference_mode()
    def _beam_texts(self, items, num_beams, max_new_tokens, temperature):
        """items: [(image, question, object_crops, images_long, objects_long)] -> decoded best hypotheses"""
        reqs = []
        for image, question, crops, il, ol in items:
            img, crops = self._pixels(image, crops)
            reqs.append((self._prompt_ids(question), img, crops, il, ol))
        outs = self.engine.generate_batch(reqs, max_new_tokens, self.eos, temperature=temperature, num_beams=num_beams,
                                          length_penalty=self.length_penalty, early_stopping=self.early_stopping)
        return [self._answer_text(out) for out in outs]

    def free_form_inference_batch(self, images, questions, max_new_tokens=200, originals=None, temperature=0, top_p=None, num_beams=1):
        """free_form_inference for several (image, question) pairs in ONE continuous-batched decode (not in the reference,
        which answers one image at a time, vstar_bench_eval.py:196): same prompt, stop string and post-processing per
        sample; each decode step reads the 7B weights once for the whole batch.  originals: the un-padded images the padded
        `images` were made from; with `use_device_images` the pixels are then produced on the GPU (bit-identical).
        temperature / top_p as in free_form_inference; each request takes one seed from torch's default generator, in order.
        num_beams > 1: beam search per request as in free_form_inference, all requests in one decode."""
        sample = temperature is not None and temperature > 0
        if sample:
            check_sampling(self.top_k, top_p)
        if num_beams != 1:
            if originals is not None and self._img_src is not None:
                images = [self.device_pixels(o, None)[0] for o in originals]
            return self._beam_texts([(im, q, None, None, None) for im, q in zip(images, questions)], num_beams, max_new_tokens,
                                    temperature)
        reqs = []
        for k, (image, question) in enumerate(zip(images, questions)):
            ids = self._prompt_ids(question)
            if originals is not None and self._img_src is not None:
                img, _ = self.device_pixels(originals[k], None)
            else:
                img, _ = self._pixels(image, None)
            reqs.append((ids, img, None, None, None))
        outs = self.engine.generate_batch(reqs, max_new_tokens, self.eos, stop_ids=self._stop_ids(),
                                          temperature=temperature if sample else 0, top_k=self.top_k, top_p=top_p,
                                          seeds=draw_seeds(len(reqs)) if sample else None)
        return [self._answer_text(out) for out in outs]

    def _prompt_ids(self, question):
        """ids of the v1 conversation prompt with the image token before `question` (vstar_bench_eval.py:79-85)"""
        return tokenizer_image_object_token(build_prompt_v1(DEFAULT_IMAGE_TOKEN + "\n" + question), self.tokenizer)

    def _stop_ids(self):
        """ids of the v1 stop string "</s>" without the tokenizer's bos (KeywordsStoppingCriteria)"""
        kw = self.tokenizer("</s>").input_ids
        if len(kw) > 1 and kw[0] == self.tokenizer.bos_token_id:
            kw = kw[1:]
        return kw

    def _answer_text(self, out):
        """new token ids -> answer text: decoded without special tokens, the stop string cut off, stripped"""
        stop_str = "</s>"
        text = self.tokenizer.batch_decode([out], skip_special_tokens=True)[0].strip()
        if text.endswith(stop_str):
            text = text[:-len(stop_str)]
        return text.strip()

    @torch.inference_mode()
    def free_form_inference_stream(self, items, max_new_tokens=200, slots=16, temperature=0, top_p=None, num_beams=1, kv_pages=None,
                                   kv_swap_pages=None, prefill_chunk=None):
        """free_form_inference for many items on one decode stream (VQAEngine.decode_stream): items are (image, question,
        object_crops, images_long, objects_long); yields (index, text) as each answer completes, with the prompt, stop string
        and post-processing of free_form_inference.  The next item is admitted whenever a slot frees, so up to `slots` answers
        decode together however much their lengths differ.  As in free_form_inference, an answer whose prompt plus
        max_new_tokens would pass the 2048 positions of the RoPE tables gets the positions that are left.
        temperature > 0 samples every item with top_k = self.top_k and top_p; the items take one seed each from torch's
        default generator, in item order, before the first admission (so torch.manual_seed(s) reproduces a call, and a call
        equals free_form_inference of each item in order after the same seed).  num_beams = k > 1 beam-searches every item
        with self.length_penalty / self.early_stopping on k slots; an item is admitted when k slots are free.
        kv_pages = N: a paged stream (VQAEngine.decode_stream) whose pool of N pages holds the KV rows; an item is then
        admitted when its slots and the pages it reserves are free, and `slots` bounds the answers decoding at a time.
        kv_swap_pages = M (with kv_pages): a growing paged stream with a host swap area of M pages; an item is then admitted
        by kv_pages.GrowingPool's rule, taking the pages it writes as it writes them.  prefill_chunk = C (with kv_pages): admitted
        prompts are prefilled C rows per step alongside the running answers (DecodeStream)."""
        reqs = [(self._prompt_ids(question), image, crops, il, ol) for image, question, crops, il, ol in items]
        paged = {} if kv_pages is None else dict(kv_pages=int(kv_pages))
        if kv_swap_pages is not None:
            paged["kv_swap_pages"] = int(kv_swap_pages)
        if prefill_chunk is not None:
            paged["prefill_chunk"] = prefill_chunk
        if (temperature is None or not temperature > 0) and num_beams == 1:
            answers = self._decode_stream(reqs, int(max_new_tokens), int(slots), **paged)
        else:
            answers = self._decode_stream(reqs, int(max_new_tokens), int(slots), settings=self._stream_settings(len(reqs), temperature,
                                                                                                            top_p, num_beams), **paged)
        for i, out in answers:
            yield i, self._answer_text(out)

    def _stream_settings(self, n, temperature, top_p, num_beams):
        """DecodeStream.admit keywords of n sampled or beam requests, validated and seeded as free_form_inference does"""
        if num_beams != 1:
            check_beams(num_beams, self.early_stopping)
            if temperature is not None and temperature > 0:
                raise NotImplementedError("num_beams > 1 with temperature > 0 (HF beam_sample) is not implemented")
            return [dict(num_beams=num_beams, length_penalty=self.length_penalty, early_stopping=self.early_stopping)] * n
        top_k, top_p = check_sampling(self.top_k, top_p)
        return [dict(temperature=temperature, top_k=top_k, top_p=top_p, seed=s) for s in draw_seeds(n)]

    def _decode_stream(self, reqs, max_new_tokens, slots, settings=None, kv_pages=None, kv_swap_pages=None, prefill_chunk=None):
        """(prompt ids, image, object_crops, images_long, objects_long) requests -> (index, new token ids) as each ends, on one
        AnswerSession with min(slots, len(reqs) * num_beams) slots and the positions of the call's largest request, admitting
        the requests in order.  settings: per request, DecodeStream.admit's generation keywords (None: greedy); kv_pages: a paged
        stream of that many pages; kv_swap_pages: growing, with that swap area; prefill_chunk: prompts prefilled that many rows
        per step"""
        if not reqs:
            return
        need = settings[0].get("num_beams", 1) if settings else 1
        prompts = [AnswerSession.prompt(self.engine, r, max_new_tokens) for r in reqs]
        positions = min(self.engine.MAX_POSITIONS, max(p.length + p.budget for p in prompts))
        session = self.answer_session(max_new_tokens, min(slots, len(reqs) * need), positions, num_beams=need, kv_pages=kv_pages,
                                      kv_swap_pages=kv_swap_pages, prefill_chunk=prefill_chunk)
        nxt = 0

        def admit():
            nonlocal nxt
            while nxt < len(reqs) and session.fits(prompts[nxt]):
                session.admit(nxt, prompts[nxt], **({} if settings is None else settings[nxt]))
                nxt += 1

        try:
            session.refuse(prompts, "the largest request of this call")
            admit()
            remaining = len(reqs)
            while remaining:
                for i, out in session.step_tokens():
                    remaining -= 1
                    yield i, out
                admit()
        finally:
            session.close()

    def answer_session(self, max_new_tokens, slots, max_positions=None, num_beams=1, kv_pages=None, kv_swap_pages=None,
                       prefill_chunk=None):
        """-> an AnswerSession: free_form_inference's answers on one decode stream of `slots` slots and `max_positions` positions
        per request (None: engine.MAX_POSITIONS), which takes requests while it runs.  A contiguous stream (kv_pages None) holds
        slots * max_positions KV rows whatever its requests need: at max_positions = engine.MAX_POSITIONS (2048) that is about
        1.6 GB per slot at 7B in bf16 or fp16 (32 layers * 2048 rows * 3 * 4096 values), so a long-lived session wants kv_pages,
        whose pool is what it says.  kv_swap_pages / prefill_chunk as in free_form_inference_stream; num_beams: the beams of
        every request"""
        return AnswerSession(self, max_new_tokens, slots, self.engine.MAX_POSITIONS if max_positions is None else max_positions,
                             num_beams, kv_pages, kv_swap_pages, prefill_chunk)

    def _choice_item(self, image, question, options, object_crops, images_long, objects_long):
        qs = DEFAULT_IMAGE_TOKEN + "\n" + question
        q_ids = tokenizer_image_object_token(build_prompt_v1(qs), self.tokenizer)
        opt_ids = []
        for option in options:
            full = tokenizer_image_object_token(build_prompt_v1(qs, option), self.tokenizer)
            opt_ids.append(full[len(q_ids):])
        img, crops = self._pixels(image, object_crops)
        return (q_ids, opt_ids, img, crops, images_long, objects_long)

    @torch.inference_mode()
    def multiple_choices_inference(self, image, question, options, object_crops=None, images_long=None, objects_long=None):
        item = self._choice_item(image, question, options, object_crops, images_long, objects_long)
        return self.engine.option_losses_batch([item])[0][1]

    @torch.inference_mode()
    def multiple_choices_inference_batch(self, requests):
        """requests: [(image, question, options, object_crops, images_long, objects_long)] -> [chosen option index].
        Not in the reference (one sample at a time, vstar_bench_eval.py:257): same per-sample result, batched execution."""
        items = [self._choice_item(*r) for r in requests]
        return [c for _, c in self.engine.option_losses_batch(items)]


class AnswerSession:
    """free_form_inference's answers on one decode stream that takes requests while it runs (VQA_LLM.answer_session): the
    admission rule, per-request budget, stop ids and text post-processing that free_form_inference_stream and
    seal.answer_open_stream share.  A request is a `prompt` (its ids, pixels, spliced length and budget); fits(p) says whether
    its slots and pages are free now, admit(key, p, **settings) starts it (DecodeStream.admit's generation keywords), and
    step() runs one decode step -> [(key, answer text)] of the requests that ended (step_tokens: their new token ids).
    `busy` while an admitted request has not been returned; close() frees the stream."""

    Prompt = namedtuple("Prompt", "ids image object_crops images_long objects_long length budget")

    @staticmethod
    def prompt(engine, request, max_new_tokens):
        """(prompt ids, image, object_crops, images_long, objects_long) -> Prompt with the spliced length T and generate()'s
        budget min(max_new_tokens, 2048 - T) new tokens"""
        ids, image, crops, il, ol = request
        T = engine.spliced_length(ids, 0 if crops is None else len(crops), il, ol)
        return AnswerSession.Prompt(ids, image, crops, il, ol, T, max(1, min(max_new_tokens, engine.MAX_POSITIONS - T)))

    def __init__(self, llm, max_new_tokens, slots, max_positions, num_beams=1, kv_pages=None, kv_swap_pages=None, prefill_chunk=None):
        if num_beams > slots:
            raise ValueError(f"num_beams = {num_beams} needs {num_beams} slots, got slots = {slots}")
        self.llm, self.max_new_tokens, self.need = llm, int(max_new_tokens), num_beams
        self.kv_pages, self.kv_swap_pages = kv_pages, kv_swap_pages
        chunk = {} if prefill_chunk is None else dict(prefill_chunk=prefill_chunk)
        self.stream = llm.engine.decode_stream(slots, max_positions, llm.eos, kv_pages=kv_pages, kv_swap_pages=kv_swap_pages, **chunk)
        # beam hypotheses end at eos alone, as in free_form_inference(num_beams > 1)
        self.stop_ids = None if num_beams > 1 else llm._stop_ids()
        self._keys = {}                                  # stream request id -> key, until returned

    def request(self, item):
        """item (image, question, object_crops, images_long, objects_long) -> its Prompt"""
        image, question, crops, il, ol = item
        return self.prompt(self.llm.engine, (self.llm._prompt_ids(question), image, crops, il, ol), self.max_new_tokens)

    def refuse(self, prompts, what):
        """ValueError naming `what` when the pool, or a growing stream's swap area, cannot hold one of the prompts however
        empty it is (checked before any launch for them)"""
        pages = self.stream.pages
        if pages is None:
            return
        if any(pages.need(p.length, p.budget, self.need) > pages.n_pages for p in prompts):
            raise ValueError(f"kv_pages = {self.kv_pages} cannot hold {what}")
        if self.stream.growing and any(pages.need(p.length, p.budget, self.need) > pages.swap_pages for p in prompts):
            raise ValueError(f"kv_swap_pages = {self.kv_swap_pages} cannot hold {what}")

    def fits(self, p):
        """whether p's slots and pages are free now (a growing stream: kv_pages.GrowingPool's admission rule)"""
        stream, pages = self.stream, self.stream.pages
        rows = stream.free_rows(self.need)
        if rows is None:
            return False
        if stream.growing:
            return pages.can_admit(rows, p.length, p.budget)
        return pages is None or pages.need(p.length, p.budget, self.need) <= pages.free_pages

    def admit(self, key, p, **settings):
        img, crops = self.llm._pixels(p.image, p.object_crops)
        r = self.stream.admit((p.ids, img, crops, p.images_long, p.objects_long), p.budget, stop_ids=self.stop_ids, **settings)
        self._keys[r.id] = key

    @property
    def busy(self):
        return bool(self._keys)

    def step_tokens(self):
        return [(self._keys.pop(r.id), out) for r, out in self.stream.step()]

    def step(self):
        return [(key, self.llm._answer_text(out)) for key, out in self.step_tokens()]

    def close(self):
        self.stream.close()
        self._keys = {}
