"""`VSM` — drop-in mirror of the reference's `visual_search.VSM` wrapper (/root/reference/visual_search.py:142-225)
on top of the sm_90a engine: host-side prompt building / tokenisation / image preprocessing, the batched engine call,
and the per-mode post-processing with the reference's return conventions.

Also hosts the checkpoint reader for the HF key layout (SURVEY.md §8f-3) and the synthetic tokenizer used when no
checkpoint/tokenizer exists (offline benches and tests).
"""
from __future__ import annotations

import glob
import json
import os
import zlib

import numpy as np
import torch

from . import ops
from .config import VSMConfig, IMAGE_TOKEN_INDEX
from .engine import VSMEngine, VSMWeights
from .image import GpuImagePipeline
from .records import pyramid_rects, record_floats
from .visual_search import (DEFAULT_IM_END_TOKEN, DEFAULT_IM_START_TOKEN, DEFAULT_IMAGE_TOKEN, Heatmap, CudaScorer, _NodeEval)

BF = torch.bfloat16
CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)

LLAVA_V1_SYSTEM = ("A chat between a curious human and an artificial intelligence assistant. "
                   "The assistant gives helpful, detailed, and polite answers to the human's questions.")


LLAVA_LLAMA_2_SYSTEM = ("You are a helpful language and vision assistant. You are able to understand the visual content that the user "
                        "provides, and assist the user with a variety of tasks using natural language.")


def build_prompt(question, conv_type="llava_v1", use_mm_start_end=True):
    """visual_search.py:176-184 + conversation.py:355-365 (conv_llava_v1: SeparatorStyle.TWO, sep=' ', sep2='</s>')."""
    prompt = DEFAULT_IMAGE_TOKEN + "\n" + question
    if use_mm_start_end:
        prompt = prompt.replace(DEFAULT_IMAGE_TOKEN, DEFAULT_IM_START_TOKEN + DEFAULT_IMAGE_TOKEN + DEFAULT_IM_END_TOKEN)
    if conv_type == "llava_llama_2":
        # conversation.py conv_llava_llama_2 (SeparatorStyle.LLAMA_2, sep "<s>", sep2 "</s>"): the system prompt is wrapped in
        # <<SYS>> and folded into the first [INST] block; the empty assistant turn adds nothing; leading "<s>" is stripped
        sys_ = "<<SYS>>\n" + LLAVA_LLAMA_2_SYSTEM + "\n<</SYS>>\n\n"
        return "[INST] " + sys_ + prompt + " [/INST]"
    if conv_type != "llava_v1":
        raise ValueError(f"unknown conv_type {conv_type!r} (visual_search.py:48: llava_v1 | llava_llama_2)")
    return LLAVA_V1_SYSTEM + " " + "USER" + ": " + prompt + " " + "ASSISTANT" + ":"


def tokenizer_image_token(prompt, tokenizer, image_token_index=IMAGE_TOKEN_INDEX):
    """VisualSearch/model/llava/mm_utils.py:19-44, reused verbatim in behaviour (defines T and the 255 offset)."""
    prompt_chunks = [tokenizer(chunk).input_ids for chunk in prompt.split("<image>")]

    def insert_separator(X, sep):
        return [ele for sublist in zip(X, [sep] * len(X)) for ele in sublist][:-1]

    input_ids = []
    offset = 0
    if len(prompt_chunks) > 0 and len(prompt_chunks[0]) > 0 and prompt_chunks[0][0] == tokenizer.bos_token_id:
        offset = 1
        input_ids.append(prompt_chunks[0][0])
    for x in insert_separator(prompt_chunks, [image_token_index] * (offset + 1)):
        input_ids.extend(x[offset:])
    return input_ids


class SyntheticTokenizer:
    """Stand-in when no sentencepiece model exists offline: deterministic hash-word tokenizer with the special tokens
    of the VSM vocabulary (32000 Llama + [PAD] + [LOC] + <im_start> + <im_end>, VisualSearch/train.py:141-148)."""
    bos_token_id, eos_token_id, unk_token_id = 1, 2, 0

    def __init__(self, cfg: VSMConfig, pad_to=None):
        self.cfg = cfg
        self.loc = cfg.loc_token_idx
        self.im_start, self.im_end = cfg.vocab - 2, cfg.vocab - 1
        self.hi = min(cfg.vocab - 24, 31990)
        self.pad_to = pad_to

    def _word(self, w):
        return 3 + zlib.crc32(w.encode()) % (self.hi - 3)

    def __call__(self, text, add_special_tokens=True):
        ids = [self.bos_token_id] if add_special_tokens else []
        for tok in text.replace(DEFAULT_IM_START_TOKEN, " <im_start> ").replace(DEFAULT_IM_END_TOKEN, " <im_end> ").replace("[LOC]", " [LOC] ").split():
            ids.append({"<im_start>": self.im_start, "<im_end>": self.im_end, "[LOC]": self.loc}.get(tok, None) or self._word(tok))

        class _R:
            pass

        r = _R()
        r.input_ids = ids
        return r

    def batch_decode(self, ids, skip_special_tokens=True):
        return [" ".join(f"w{int(t)}" for t in row if not (skip_special_tokens and int(t) in (0, 1, 2))) for row in ids]


# ----------------------------------------------------------------------------------------------------------------
# host image preprocessing (visual_search.py:186-194).  PIL bicubic like the HF processors the reference uses, into
# PINNED staging buffers so the H2D copy is asynchronous.
# ----------------------------------------------------------------------------------------------------------------
def expand2square(pil_img, background_color):
    # VisualSearch/utils/utils.py:28-39 : paste at TOP-LEFT, pad bottom/right
    from PIL import Image
    width, height = pil_img.size
    if width == height:
        return pil_img
    side = max(width, height)
    result = Image.new(pil_img.mode, (side, side), background_color)
    result.paste(pil_img, (0, 0))
    return result


_MEAN = np.array(CLIP_MEAN, np.float32)
_STD = np.array(CLIP_STD, np.float32)


def _normalize_into(arr_u8, dst):
    x = arr_u8.astype(np.float32) * np.float32(1 / 255.0)
    x = (x - _MEAN) / _STD
    dst.copy_(torch.from_numpy(np.ascontiguousarray(x.transpose(2, 0, 1))))


def preprocess_clip_into(pil_img, dst, size=224):
    from PIL import Image
    bg = tuple(int(x * 255) for x in CLIP_MEAN)
    img = expand2square(pil_img.convert("RGB"), bg)
    w, h = img.size
    short = min(w, h)
    nw, nh = int(w * size / short), int(h * size / short)
    img = img.resize((nw, nh), resample=Image.BICUBIC)
    left, top = (nw - size) // 2, (nh - size) // 2
    _normalize_into(np.array(img.crop((left, top, left + size, top + size))), dst)


def preprocess_owl_into(pil_img, dst, size=768):
    from PIL import Image
    _normalize_into(np.array(pil_img.convert("RGB").resize((size, size), resample=Image.BICUBIC)), dst)


# ----------------------------------------------------------------------------------------------------------------
# checkpoint reader (HF sharded safetensors / .bin with the reference key layout)
# ----------------------------------------------------------------------------------------------------------------
from .checkpoint import open_checkpoint  # noqa: E402,F401  (safetensors -> GPU streaming reader / mmap'd .bin shards)


def config_from_hf(path) -> VSMConfig:
    j = json.load(open(os.path.join(path, "config.json")))
    cfg = VSMConfig(hidden=j["hidden_size"], n_layers=j["num_hidden_layers"], n_heads=j["num_attention_heads"],
                    intermediate=j["intermediate_size"], vocab=j["vocab_size"], rms_eps=j.get("rms_norm_eps", 1e-6),
                    owl_query_dim=j.get("out_dim", 512))
    return cfg


class VSM:
    """Same surface as the reference wrapper: `VSM(args)`, `.inference(image, question, mode)`; plus `detect_batch`."""

    def __init__(self, args=None, engine: VSMEngine = None, tokenizer=None, frontier_batch=8, draft_answer="Sure, [LOC].",
                 forced_answer_ids=None, prep="gpu"):
        if engine is None:
            # visual_search.py:143-172: tokenizer + checkpoint from args.version, CLIP tower from args.vision_tower
            if args is None or not os.path.isdir(str(args.version)):
                raise FileNotFoundError(
                    "VSM(args): args.version must be a local checkpoint directory (no network here); pass engine= / tokenizer= "
                    "for synthetic weights")
            from transformers import AutoTokenizer
            tokenizer = AutoTokenizer.from_pretrained(args.version, model_max_length=args.model_max_length, padding_side="right", use_fast=False)
            tokenizer.pad_token = tokenizer.unk_token
            cfg = config_from_hf(args.version)
            cfg.loc_token_idx = tokenizer("[LOC]", add_special_tokens=False).input_ids[0]
            main = open_checkpoint(args.version, device="cuda")
            clip = open_checkpoint(args.vision_tower, device="cuda")     # CLIP weights are not in the VSM checkpoint (merge...py:146-149)

            def get(name):
                pfx = "model.vision_tower.vision_tower."
                return clip(name[len(pfx):]) if name.startswith(pfx) else main(name)

            # cache rows per crop: the tokenizer truncates text at model_max_length; the splice adds 255 rows; the cache grows
            # on demand for generations beyond that (engine._ensure_cache)
            engine = VSMEngine(VSMWeights(cfg, get), max_tokens=min(2048, int(args.model_max_length)))
            self.conv_type, self.use_mm_start_end = args.conv_type, args.use_mm_start_end
        else:
            self.conv_type, self.use_mm_start_end = "llava_v1", True
        self.engine = engine
        self.model = engine                       # attribute name kept from the reference wrapper
        self.cfg = engine.cfg
        self.vsm_tokenizer = tokenizer if tokenizer is not None else SyntheticTokenizer(self.cfg)
        self.frontier_batch = frontier_batch
        self.scorer = CudaScorer()
        eos = getattr(self.vsm_tokenizer, "eos_token_id", 2)
        self.eos = eos
        self.draft_ids = list(self.vsm_tokenizer(draft_answer, add_special_tokens=False).input_ids) + [eos]
        self.forced_answer_ids = forced_answer_ids      # synthetic weights only: logits-processor-style forcing
        if forced_answer_ids is not None:
            self.draft_ids = list(forced_answer_ids)
        self._pinned = {}
        self.timers = dict(prep=0.0, engine=0.0)
        # prep="gpu": crops are cut + resized on the device from the resident search image (Pillow-exact integer
        # bicubic); prep="host": the reference's PIL path (kept for parity tests of the pipeline itself)
        self.prep = prep
        self.pipeline = GpuImagePipeline(engine.dev, self.cfg.clip_image, self.cfg.owl_image) if prep == "gpu" else None
        self._resident = {}          # id(PIL image) -> (PIL image, uint8 HWC device tensor)
        # crops per engine call while search images are still being uploaded (see _run); 0 = never split
        self.upload_chunk = int(os.environ.get("VSB_UPLOAD_CHUNK", "16"))
        self.h2d_bytes = 0
        self.d2h_bytes = 0
        self.vqa_max_new_tokens = 100          # max_new_tokens of VSM.inference(mode='vqa') (visual_search.py:201)
        self._host_pool = {}
        self._d2h_stream = None

    # ------------------------------------------------------------------ host prep
    def _staging(self, B):
        """pinned staging buffers of the host-prep path, one set per batch size, guarded by the event of the last H2D copy out
        of them (several prompt-length groups of the same size are launched back to back without a host sync)"""
        c = self.cfg
        slot = self._pinned.get(B)
        if slot is None:
            slot = [torch.empty((B, 3, c.clip_image, c.clip_image), dtype=torch.float32).pin_memory(),
                    torch.empty((B, 3, c.owl_image, c.owl_image), dtype=torch.float32).pin_memory(), None]
            self._pinned[B] = slot
        if slot[2] is not None:
            slot[2].synchronize()             # the copy queued by the previous user of this slot has read the buffer
        return slot

    def _prep(self, images):
        """host path: PIL crops -> (clip [B,3,224,224], owl [B,3,768,768]) bf16 on the device"""
        c = self.cfg
        B = len(images)
        slot = self._staging(B)
        pc, po = slot[0], slot[1]
        for i, im in enumerate(images):
            preprocess_clip_into(im, pc[i], c.clip_image)
            preprocess_owl_into(im, po[i], c.owl_image)
        self.h2d_bytes += pc.numel() * 4 + po.numel() * 4
        dc, do = pc.cuda(non_blocking=True), po.cuda(non_blocking=True)
        slot[2] = torch.cuda.Event()
        slot[2].record()
        ic = ops.cast_f32_bf16(dc)      # .bfloat16() of the reference (visual_search.py:189,194)
        io = ops.cast_f32_bf16(do)
        return ic, io

    def resident(self, pil_img):
        """uint8 HWC copy of a search image in HBM (uploaded once, reused by every crop of that search)"""
        key = id(pil_img)
        hit = self._resident.get(key)
        if hit is None or hit[0] is not pil_img:
            if len(self._resident) >= 64:
                self._resident.pop(next(iter(self._resident)))
            t = self.pipeline.upload(pil_img)
            self.h2d_bytes += t.numel()
            self._resident[key] = (pil_img, t)
            return t
        return hit[1]

    def release(self, pil_img=None):
        if pil_img is None:
            self._resident.clear()
        else:
            self._resident.pop(id(pil_img), None)

    def _prep_regions(self, regions):
        """regions: list of (source PIL image, bbox [x,y,w,h]) -> device pixel tensors via the GPU image pipeline"""
        if self.prep != "gpu":
            crops = [src.crop((int(b[0]), int(b[1]), int(b[0] + b[2]), int(b[1] + b[3]))) for src, b in regions]
            return self._prep(crops)
        c = self.cfg
        B = len(regions)
        ic = torch.empty((B, 3, c.clip_image, c.clip_image), dtype=BF, device=self.engine.dev)
        io = torch.empty((B, 3, c.owl_image, c.owl_image), dtype=BF, device=self.engine.dev)
        for i, (src, b) in enumerate(regions):
            self.pipeline.crop_tensors(self.resident(src), b, ic[i], io[i])
        return ic, io

    def _ids(self, question):
        prompt = build_prompt(question, self.conv_type, self.use_mm_start_end)
        return tokenizer_image_token(prompt, self.vsm_tokenizer)

    # ------------------------------------------------------------------ engine calls
    def _host_buffer(self, shape, dtype):
        """pinned host buffers for the per-batch D2H copies, recycled (page-locking per batch costs more than the copy)"""
        n = 1
        for v in shape:
            n *= int(v)
        key = (dtype, max(1024, 1 << (max(1, n) - 1).bit_length()))
        pool = self._host_pool.setdefault(key, [])
        buf = pool.pop() if pool else torch.empty((key[1],), dtype=dtype).pin_memory()
        return buf, key

    def _launch(self, regions, questions, mode, smallest=None, rec_len=None):
        """Queue the evaluation of a batch on the GPU and return at once (nothing here waits for the device).
        regions: list of (source PIL image, bbox).  smallest: per-region smallest_size => crop RECORDS are produced on the
        device (records.py) and copied to pinned host memory on a side stream; None => per-crop tensors only."""
        import time
        t0 = time.perf_counter()
        dev = self.engine.dev
        n = len(regions)
        ids_list = [self._ids(q) for q in questions]
        groups = {}
        for i, ids in enumerate(ids_list):
            groups.setdefault((len(ids), ids.index(IMAGE_TOKEN_INDEX)), []).append(i)
        pend = dict(n=n, mode=mode, regions=regions, smallest=smallest, chunks=[], rec=None, rects=None, low=[None] * n,
                    det=[None] * n)
        rec = None
        if smallest is not None:
            rects = [pyramid_rects(b, ss) for (_, b), ss in zip(regions, smallest)]
            R = record_floats(max(len(r) for r in rects))
            rec = torch.zeros((n, max(R, rec_len or 0)), dtype=torch.float32, device=dev)
            pend["rec"], pend["rects"] = rec, rects
        heat_jobs = []
        for key, members in groups.items():
            # Search images that are not resident yet cost ~1.5 ms of host time each (PIL -> pinned staging -> H2D).  Such a
            # group is cut into chunks whose engine work is launched WITHOUT waiting for the GPU (defer=True), so the host
            # converts the next chunk's images while the GPU evaluates the previous one.
            fresh = len({id(regions[i][0]) for i in members if self.prep == "gpu" and id(regions[i][0]) not in self._resident})
            step = len(members)
            if self.upload_chunk > 0 and fresh >= 4:          # (distinct images that still have to be uploaded)
                # crops of the same image next to each other: the first chunk then needs only the first few uploads
                order = {}
                for i in members:
                    order.setdefault(id(regions[i][0]), len(order))
                members = sorted(members, key=lambda i: order[id(regions[i][0])])
                # at least two chunks when several images still have to be uploaded: the first engine call starts after half of
                # the conversions instead of all of them
                step = max(2, min(self.upload_chunk, (len(members) + 1) // 2))
            for c0 in range(0, len(members), step):
                chunk = members[c0:c0 + step]
                ic, io = self._prep_regions([regions[i] for i in chunk])
                t1 = time.perf_counter()
                self.timers["prep"] += t1 - t0
                prompt = torch.tensor([ids_list[i] for i in chunk], dtype=torch.int64)
                if mode == "vqa" and self.forced_answer_ids is None:
                    # free-form answer (the cue question): nothing to draft-verify - batched exact greedy decoding
                    toks = self.engine.generate_many(prompt, ic, max_new_tokens=self.vqa_max_new_tokens, eos_token_id=self.eos)
                    out = dict(output_ids=[torch.tensor(t) for t in toks], verified=[True] * len(chunk), n_crops=len(chunk))
                    pend["chunks"].append([chunk, out, io, ic, prompt, None])
                    t0 = time.perf_counter()
                    self.timers["engine"] += t0 - t1
                    continue
                out = self.engine.inference(io, ic, prompt, self.draft_ids, eos_token_id=self.eos, mode=mode,
                                            forced_ids=self.forced_answer_ids, defer=True)
                if rec is not None:
                    heat_jobs += self._pack_chunk(out, chunk, pend)
                pend["chunks"].append([chunk, out, io, ic, prompt, None])
                t0 = time.perf_counter()
                self.timers["engine"] += t0 - t1
        if heat_jobs:
            c = self.cfg
            ops.heat_pyramids(heat_jobs, rec, 4 * c.owl_grid, 4 * c.owl_grid)
        # device -> host on a side stream: finish() waits for THIS batch only, not for whatever was queued behind it
        main = torch.cuda.current_stream()
        ready = torch.cuda.Event()
        ready.record(main)
        if self._d2h_stream is None:
            self._d2h_stream = torch.cuda.Stream(device=dev)
        keys = []
        with torch.cuda.stream(self._d2h_stream):
            self._d2h_stream.wait_event(ready)
            if rec is not None:
                buf, key = self._host_buffer(rec.shape, torch.float32)
                keys.append((key, buf))
                pend["rec_host"] = buf[:rec.numel()].view(rec.shape)
                pend["rec_host"].copy_(rec, non_blocking=True)
                rec.record_stream(self._d2h_stream)
                self.d2h_bytes += rec.numel() * 4
            for ch in pend["chunks"]:
                am = ch[1].get("_am")
                if am is not None:
                    buf, key = self._host_buffer(am.shape, am.dtype)
                    keys.append((key, buf))
                    ch[5] = buf[:am.numel()].view(am.shape)
                    ch[5].copy_(am, non_blocking=True)
                    am.record_stream(self._d2h_stream)
                    self.d2h_bytes += am.numel() * am.element_size()
            done = torch.cuda.Event()
            done.record(self._d2h_stream)
        pend["done"], pend["host_keys"] = done, keys
        self.timers["engine"] += time.perf_counter() - t0
        return pend

    def _pack_chunk(self, out, chunk, pend):
        """detections of one engine call -> record rows (device); returns the heat-map jobs of its expandable crops"""
        rec, rects = pend["rec"], pend["rects"]
        col = out["crop_of_loc"]
        B = len(chunk)
        low = out["low_res_masks"]
        seg_only = pend["mode"] == "segmentation"          # cue segmentation: the record carries the heat-map part only
        scores = boxes = None
        if col == list(range(B)):
            first = last = list(range(B))
        else:                                   # several [LOC] per answer: pred_boxes[0] / pred_mask[-1] (visual_search.py:208-211)
            first = [col.index(j) for j in range(B)]
            last = [len(col) - 1 - col[::-1].index(j) for j in range(B)]
        if not seg_only:
            scores, boxes = out["scores"], out["pred_boxes"]
            if first != list(range(B)):
                idx = torch.tensor(first, device=scores.device)
                scores, boxes = scores.index_select(0, idx).contiguous(), boxes.index_select(0, idx).contiguous()
            if chunk == list(range(chunk[0], chunk[0] + B)):
                ops.pack_detections(scores.contiguous(), boxes.contiguous(), rec, row0=chunk[0])
            else:
                tmp = torch.zeros((B, rec.shape[1]), dtype=torch.float32, device=rec.device)
                ops.pack_detections(scores.contiguous(), boxes.contiguous(), tmp)
                rec.index_copy_(0, torch.tensor(chunk, device=rec.device), tmp)
        jobs = []
        for j, i in enumerate(chunk):
            pend["low"][i] = low[last[j]]
            pend["det"][i] = (scores[j], boxes[j]) if not seg_only else None
            if rects[i]:
                bb = pend["regions"][i][1]
                x0, y0 = int(bb[0]), int(bb[1])
                jobs.append((low[last[j]], int(bb[3]), int(bb[2]), [(r[0] - x0, r[1] - y0, r[2], r[3]) for r in rects[i]], i))
        return jobs

    def _finish(self, pend):
        """wait for the batch's device->host copies, resolve the draft verification, return per-crop results:
        record mode -> list of _NodeEval; otherwise list of dicts with device tensors"""
        import time
        t0 = time.perf_counter()
        pend["done"].synchronize()
        mode, n = pend["mode"], pend["n"]
        results = [None] * n
        redo = []
        for chunk, out, io, ic, prompt, am_host in pend["chunks"]:
            self.engine.finish(out, am_host)
            for j, i in enumerate(chunk):
                if out["verified"][j]:
                    results[i] = self._slice(out, j, mode) if pend["rec"] is None else True
                else:
                    redo.append((i, io[j:j + 1], ic[j:j + 1], prompt[j:j + 1]))
        rows = pend["rec_host"].numpy() if pend["rec"] is not None else None
        for i, io1, ic1, prompt1 in redo:
            r = self._exact_single(io1, ic1, prompt1, mode)          # exact greedy decode of this crop (synchronous, rare)
            if rows is None:
                results[i] = r
                continue
            rec1 = torch.zeros((1, rows.shape[1]), dtype=torch.float32, device=self.engine.dev)
            if mode != "segmentation":
                ops.pack_detections(r["scores"].view(1, -1).contiguous(), r["boxes"].view(1, -1, 4).contiguous(), rec1)
            if pend["rects"][i]:
                bb = pend["regions"][i][1]
                x0, y0 = int(bb[0]), int(bb[1])
                ops.heat_pyramids([(r["low_res"].contiguous(), int(bb[3]), int(bb[2]),
                                    [(q[0] - x0, q[1] - y0, q[2], q[3]) for q in pend["rects"][i]], 0)], rec1,
                                  r["low_res"].shape[-2], r["low_res"].shape[-1])
            rows[i] = rec1.cpu().numpy()[0]
            pend["low"][i] = r["low_res"]
            pend["det"][i] = (r["scores"].view(-1), r["boxes"].view(-1, 4)) if mode != "segmentation" else None
            results[i] = True
        if rows is not None:
            for i in range(n):
                ev = _NodeEval.from_record(rows[i], pend["regions"][i][1], pend["smallest"][i])
                ev.low_res = pend["low"][i]
                if pend["det"][i] is not None:
                    ev.scores, ev.boxes = pend["det"][i]

                    def fetch_valid(sb=pend["det"][i]):
                        return sb[1][sb[0].view(-1) > 0.5].view(-1, 4).cpu()

                    ev.fetch_valid = fetch_valid
                results[i] = ev
            rows = None
        for key, buf in pend["host_keys"]:
            self._host_pool.setdefault(key, []).append(buf)
        self.timers["engine"] += time.perf_counter() - t0
        return results

    def _run(self, regions, questions, mode):
        """regions: list of (source PIL image, bbox) -> list (per crop) of dicts with device tensors"""
        return self._finish(self._launch(regions, questions, mode))

    def _exact_single(self, io, ic, prompt, mode):
        """draft mismatch: exact greedy decode on the KV cache, then one teacher-forced pass over the emitted ids
        (== the reference's last generate step, VSM.py:459)."""
        out_ids, _ = self.engine.generate(prompt, ic, max_new_tokens=100, eos_token_id=self.eos)
        res = dict(output_ids=torch.tensor(out_ids))
        if mode == "vqa":
            return res
        ids = torch.tensor([out_ids[:-1]], dtype=torch.int64, device=self.engine.dev)
        if self.cfg.loc_token_idx not in out_ids:
            raise RuntimeError("no [LOC] token generated (reference: IndexError at visual_search.py:209-211)")
        out = self.engine.model_forward(io, ic, ids, mode=mode)
        out["output_ids"] = [res["output_ids"]]
        return self._slice(out, 0, mode)

    @staticmethod
    def _slice(out, j, mode):
        r = dict(output_ids=out["output_ids"][j])
        if mode == "vqa":
            return r
        locs = [k for k, b in enumerate(out["crop_of_loc"]) if b == j]
        r["low_res"] = out["low_res_masks"][locs[-1]]             # pred_mask[-1]  (visual_search.py:211, :225)
        if mode == "detection":
            f = locs[0]                                           # pred_boxes[0] / pred_logits[0]
            r["scores"] = out["scores"][f]
            r["logits"] = out["pred_logits"][f]
            r["boxes"] = out["pred_boxes"][f]                     # owl_heads returns boxes per (crop, query) entry
        return r

    # ------------------------------------------------------------------ public API
    @torch.inference_mode()
    def inference(self, image, question, mode="segmentation"):
        """visual_search.py:174-225.  'segmentation' -> Heatmap-backed fp32 tensor [h,w] on GPU (>= 0);
        'vqa' -> str; 'detection' -> (boxes [P,4] CPU, scores [P,1] CPU, heatmap [h,w] GPU)."""
        r = self._run([(image, [0, 0, image.width, image.height])], [question], mode)[0]
        if self.prep == "gpu":
            self.release(image)           # a crop handed in by a caller is not a long-lived search image
        if mode == "vqa":
            input_len = len(self._ids(question))
            text = self.vsm_tokenizer.batch_decode(r["output_ids"][input_len:].view(1, -1), skip_special_tokens=True)[0]
            return text.replace("\n", "").replace("  ", " ").strip()
        h, w = image.height, image.width
        heat = self.scorer.from_low_res(r["low_res"], h, w)
        if mode == "segmentation":
            return heat.map
        return r["boxes"].cpu(), r["scores"].view(-1, 1).cpu(), heat.map

    @torch.inference_mode()
    def inference_many(self, regions, questions, mode, smallest_sizes=None):
        """`inference` for several (search image, bbox) crops in ONE batched engine call - used by the search controller for
        the weak-cue branch of many lock-step searches (visual_search.py:427-443 runs these one node at a time).
        'vqa' -> list of str; 'segmentation' -> list of Heatmap (clamped H x W map on the GPU + statistics), or - when the
        searches' smallest_sizes are given - list of _NodeEval whose `.pyramid` holds the statistics and quad-tree sums of the cue
        map (built on the device like the detection records: no H x W map, no per-node host sync)."""
        if mode == "segmentation" and smallest_sizes is not None:
            return self._finish(self._launch(regions, questions, "segmentation", smallest=list(smallest_sizes)))
        rs = self._run(regions, questions, mode)
        if mode == "vqa":
            out = []
            for r, q in zip(rs, questions):
                input_len = len(self._ids(q))
                text = self.vsm_tokenizer.batch_decode(r["output_ids"][input_len:].view(1, -1), skip_special_tokens=True)[0]
                out.append(text.replace("\n", "").replace("  ", " ").strip())
            return out
        assert mode == "segmentation"
        return [self.scorer.from_low_res(r["low_res"], int(b[3]), int(b[2])) for r, (_, b) in zip(rs, regions)]

    def detect_batch(self, images, questions):
        """PIL crops in, see detect_regions"""
        return self.detect_regions([(im, [0, 0, im.width, im.height]) for im in images], questions)

    cue_records = True          # inference_many(mode="segmentation", smallest_sizes=...) answers with crop records (see there)

    @torch.inference_mode()
    def detect_regions_launch(self, regions, questions, smallest_sizes, rec_len=None, mode="detection"):
        """Asynchronous batched detection-mode evaluation for the search controller: regions = [(search image, bbox)].
        smallest_sizes[i] = the search's smallest_size (decides whether crop i will ever be split, i.e. needs the heat-map
        part of its record).  rec_len: record length in floats when the caller needs a common one (sharded frontier: the
        all-gather wants the same record size on every rank).  mode="segmentation": the cue segmentation of the weak-cue branch -
        the record then carries only the heat-map part (statistics + quad-tree sums).  Returns a handle for detect_regions_finish."""
        return self._launch(regions, questions, mode, smallest=list(smallest_sizes), rec_len=rec_len)

    @torch.inference_mode()
    def detect_regions_finish(self, handle):
        """-> [_NodeEval] built from the batch's crop records (one D2H per batch, issued at launch on a side stream)"""
        return self._finish(handle)

    def detect_regions(self, regions, questions, smallest_sizes=None):
        """synchronous form.  Without smallest_sizes every crop gets the heat-map statistics and the sums of its four children
        (enough for one expansion; deeper levels need the search's smallest_size)."""
        if smallest_sizes is None:
            smallest_sizes = [max(1, min(int(b[2]), int(b[3])) // 2) for _, b in regions]
        return self.detect_regions_finish(self.detect_regions_launch(regions, questions, smallest_sizes))


# ----------------------------------------------------------------------------------------------------------------
# model-loading API mirror (SURVEY.md §8b): VSMForCausalLM.from_pretrained / .inference / .model_forward
# ----------------------------------------------------------------------------------------------------------------
class _VisionTowerHandle:
    """what `vsm_model.get_model().get_vision_tower()` hands to the reference wrapper (visual_search.py:160-162)"""

    def __init__(self):
        self.image_processor = None

    def cuda(self):
        return self

    def to(self, *a, **k):
        return self


class _Cfg:
    pass


class VSMForCausalLM:
    """Drop-in for VisualSearch/model/VSM.py:162-553 (inference paths only) on the sm_90a engine."""

    def __init__(self, engine: VSMEngine, vision_tower_name="openai/clip-vit-large-patch14"):
        self.engine = engine
        self.cfg = engine.cfg
        self.loc_token_idx = engine.cfg.loc_token_idx
        self.config = _Cfg()
        self.config.vision_tower = vision_tower_name
        self.config.mm_vision_tower = vision_tower_name
        self.config.vocab_size = engine.cfg.vocab
        self._tower = _VisionTowerHandle()

    @classmethod
    def from_pretrained(cls, version, low_cpu_mem_usage=True, vision_tower="openai/clip-vit-large-patch14", loc_token_idx=None,
                        torch_dtype=torch.bfloat16, device_map="cuda", is_eval=True, **kwargs):
        """visual_search.py:157-159.  `version` = local checkpoint dir (HF shards, key layout of
        merge_lora_weights_and_save_hf_model.py:143-151); CLIP weights come from the `vision_tower` directory."""
        if torch_dtype != torch.bfloat16:
            raise NotImplementedError("the sm_90a kernels compute in bf16 (the reference loads the VSM in bf16 too)")
        cfg = config_from_hf(version)
        if loc_token_idx is not None:
            cfg.loc_token_idx = int(loc_token_idx)
        device = "cuda" if device_map in ("cuda", "auto") else device_map
        main = open_checkpoint(version, device=device)
        clip = open_checkpoint(vision_tower, device=device)

        def get(name):
            pfx = "model.vision_tower.vision_tower."
            return clip(name[len(pfx):]) if name.startswith(pfx) else main(name)

        return cls(VSMEngine(VSMWeights(cfg, get, device=device)), vision_tower)

    # -- HF-style accessors used by the reference wrapper
    def get_model(self):
        return self

    def initialize_vision_modules(self, cfg):
        return None                       # CLIP is part of the engine weights already

    def get_vision_tower(self):
        return self._tower

    def eval(self):
        return self

    def _ids_rows(self, ids_1d, T, img_pos):
        c = self.cfg
        return [(k - 1) + c.clip_tokens - 1 for k in (ids_1d == c.loc_token_idx).nonzero().flatten().tolist()]

    @torch.inference_mode()
    def model_forward(self, images, images_clip, input_ids, original_size_list=None, label_list=None, inference=True, **_unused):
        """VSM.py:201-364 with inference=True (batch of teacher-forced samples sharing one length)"""
        assert inference, "training losses are outside the hot path"
        out = self.engine.model_forward(images.to(torch.bfloat16), images_clip.to(torch.bfloat16), input_ids)
        sizes = original_size_list if original_size_list is not None else [tuple(l.shape) for l in label_list]
        pred_masks = []
        for b in range(input_ids.shape[0]):
            locs = [k for k, cb in enumerate(out["crop_of_loc"]) if cb == b]
            h, w = sizes[b]
            pred_masks.append(torch.stack([ops.heatmap(out["low_res_masks"][k].contiguous(), int(h), int(w), clamp=False, with_stats=False)[0] for k in locs]))
        return {"pred_masks": pred_masks, "gt_masks": None, "pred_logits": out["pred_logits"].unsqueeze(-1),
                "pred_boxes": out["pred_boxes"], "gt_bboxes": None}

    @torch.inference_mode()
    def inference(self, images_clip, images, input_ids, resize_list, original_size_list, max_new_tokens=32, tokenizer=None, mode="vqa"):
        """VSM.py:438-553: greedy generate, then (mode != 'vqa') the seg / det branches.  Returns
        (output_ids [1,L] | None, [pred_masks [n_loc,h,w]] | None, {'pred_logits','pred_boxes'} | None)."""
        assert mode in ["vqa", "segmentation", "detection"]
        assert input_ids.shape[0] == 1, "the reference wrapper evaluates one crop per call"
        eos = getattr(tokenizer, "eos_token_id", 2) if tokenizer is not None else 2
        ic = images_clip.to(torch.bfloat16)
        out_ids, _ = self.engine.generate(input_ids.cpu(), ic, max_new_tokens=max_new_tokens, eos_token_id=eos)
        output_ids = torch.tensor([out_ids], dtype=torch.int64, device=input_ids.device)
        if mode == "vqa":
            return output_ids, None, None
        if self.loc_token_idx not in out_ids:
            # the reference returns empty lists here and its wrapper then fails with IndexError (visual_search.py:209-211)
            return None, [], None
        ids = torch.tensor([out_ids[:-1]], dtype=torch.int64, device=self.engine.dev)     # last generate step's input (VSM.py:459)
        out = self.engine.model_forward(images.to(torch.bfloat16), ic, ids, mode=mode)
        h, w = original_size_list[0]
        pm = torch.stack([ops.heatmap(out["low_res_masks"][k].contiguous(), int(h), int(w), clamp=False, with_stats=False)[0]
                          for k in range(out["low_res_masks"].shape[0])])
        if mode == "segmentation":
            return None, [pm], None
        return None, [pm], {"pred_logits": out["pred_logits"].unsqueeze(-1), "pred_boxes": out["pred_boxes"]}
