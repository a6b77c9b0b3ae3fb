"""Drop-in mirror of /root/reference/visual_search.py for the guided visual-search hot path.

Same public names and conventions (SURVEY.md §8b): `parse_args`, `VSM`, `VSM.inference(image, question, mode)`,
`visual_search(...) -> (final_step, path_length, search_successful, all_valid_boxes)`, plus the INT geometry helpers.

What is different underneath (H100-first):
  * the controller is ITERATIVE (the reference recurses once per expanded node and dies at ~990 nodes, SURVEY.md §3B)
    but pops the very same `queue.PriorityQueue` / `Prioritize` objects in the very same push/pop sequence, so the
    expansion order (including heapq tie behaviour) is the reference's;
  * frontier nodes are evaluated SPECULATIVELY in batches (each node's outputs are a pure function of its crop) and
    committed strictly in pop order; speculative work is simply dropped when the search ends early;
  * several searches can run in lock-step (`visual_search_many`) so their frontiers share one GPU batch, or be admitted
    continuously into one controller (`SearchController.stream`, used by the search-only evaluation `main`);
  * every crop evaluation comes back as ONE fixed-size record (records.py): best score/box, the boxes above 0.5, the
    heat-map statistics and the sums of the normalised map over the crop's quad-tree descendants — computed on the GPU
    straight from the 192 x 192 low-res mask.  Committing a node is then pure host arithmetic on records of the node
    and its ancestors: no H x W map is written, copied (visual_search.py:448) or re-read per expansion, and nothing
    synchronises with the GPU between the arrival of a batch and the launch of the next one;
  * batches are PIPELINED: while one frontier batch runs on the GPU the controller commits the previous one and
    launches the next (`depth` batches in flight), so the GPU does not idle across the host's commit phase.
"""
from __future__ import annotations

import argparse
import functools
import json
import os
import sys
from queue import PriorityQueue

import numpy as np
import torch

from . import ops

# ---------------------------------------------------------------------------------------------------------------
# CLI / constants (visual_search.py:28-52; VisualSearch/utils/utils.py:7-12)
# ---------------------------------------------------------------------------------------------------------------
IGNORE_INDEX = -100
IMAGE_TOKEN_INDEX = -200
DEFAULT_IMAGE_TOKEN = "<image>"
DEFAULT_IM_START_TOKEN = "<im_start>"
DEFAULT_IM_END_TOKEN = "<im_end>"

DETECTION_QUESTION = "Please locate the {} in this image."
CUE_QUESTION = ("According to the common sense knowledge and possible visual cues, what is the most likely location of "
                "the {} in the image?")


def parse_args(args):
    parser = argparse.ArgumentParser(description="Visual Search Evaluation")
    parser.add_argument("--version", default="craigwu/seal_vsm_7b")
    parser.add_argument("--benchmark-folder", default="vstar_bench", type=str)
    parser.add_argument("--visualization", action="store_true", default=False)
    parser.add_argument("--output_path", default="", type=str)
    parser.add_argument("--confidence_low", default=0.3, type=float)
    parser.add_argument("--confidence_high", default=0.5, type=float)
    parser.add_argument("--target_cue_threshold", default=6.0, type=float)
    parser.add_argument("--target_cue_threshold_decay", default=0.7, type=float)
    parser.add_argument("--target_cue_threshold_minimum", default=3.0, type=float)
    parser.add_argument("--minimum_size_scale", default=4.0, type=float)
    parser.add_argument("--minimum_size", default=224, type=int)
    parser.add_argument("--model_max_length", default=512, type=int)
    parser.add_argument("--vision-tower", default="openai/clip-vit-large-patch14", type=str)
    parser.add_argument("--use_mm_start_end", action="store_true", default=True)
    parser.add_argument("--conv_type", default="llava_v1", type=str, choices=["llava_v1", "llava_llama_2"])
    # scheduling of `main` (not in the reference, which runs one search at a time); none of these changes a result
    parser.add_argument("--searches-in-flight", default=32, type=int,
                        help="searches kept active at once; the next target is admitted when one ends (1 = the reference's order)")
    parser.add_argument("--search-batch", default=64, type=int, help="frontier crops per VSM call")
    parser.add_argument("--trajectory-json", default=None, type=str,
                        help="write one record per target (expanded boxes and scores, final box, IoU, latency) to this file")
    return parser.parse_args(args)


# ---------------------------------------------------------------------------------------------------------------
# INT geometry (visual_search.py:227-253, :277-283) — host code, bit-exact by construction
# ---------------------------------------------------------------------------------------------------------------
def refine_bbox(bbox, image_width, image_height):
    bbox[0] = max(0, bbox[0])
    bbox[1] = max(0, bbox[1])
    bbox[2] = min(bbox[2], image_width - bbox[0])
    bbox[3] = min(bbox[3], image_height - bbox[1])
    return bbox


# split_4subpatches / get_sub_patches (visual_search.py:234-253) live in records.py (the record layout is defined by the same
# quad-tree geometry) and are re-exported here under the reference's names
from .records import expandable, get_sub_patches, parse_record, pyramid_rects, split_4subpatches  # noqa: E402,F401


def iou(bbox1, bbox2):
    x1 = max(bbox1[0], bbox2[0])
    y1 = max(bbox1[1], bbox2[1])
    x2 = min(bbox1[0] + bbox1[2], bbox2[0] + bbox2[2])
    y2 = min(bbox1[1] + bbox1[3], bbox2[1] + bbox2[3])
    inter_area = max(0, x2 - x1) * max(0, y2 - y1)
    return inter_area / (bbox1[2] * bbox1[3] + bbox2[2] * bbox2[3] - inter_area)


@functools.total_ordering
class Prioritize:
    # visual_search.py:378-389: compares priority only; ties are resolved by heapq's sift order
    def __init__(self, priority, item):
        self.priority = priority
        self.item = item

    def __eq__(self, other):
        return self.priority == other.priority

    def __lt__(self, other):
        return self.priority < other.priority


# ---------------------------------------------------------------------------------------------------------------
# heat-map scoring on the GPU (visual_search.py:255-275, :420-427, :453-462)
# ---------------------------------------------------------------------------------------------------------------
class Heatmap:
    """A clamped full-resolution target-cue map resident on the GPU with its (max, min, sum)."""
    __slots__ = ("map", "stats", "h", "w", "_stats_host")

    def __init__(self, map_, stats, h, w):
        self.map, self.stats, self.h, self.w = map_, stats, h, w
        self._stats_host = None

    def host_stats(self):
        if self._stats_host is None:
            self._stats_host = self.stats.cpu().numpy()
        return self._stats_host

    def normalized(self):
        """normalize_score(...) as a [h,w,1] fp32 numpy array (what the reference stores in search_path)"""
        mx, mn = float(self.host_stats()[0]), float(self.host_stats()[1])
        m = self.map.cpu().numpy()
        m = (m - np.float32(mn)) / np.float32(mx - mn) if mx != mn else m * 0
        return m.reshape(self.h, self.w, 1)

    def __array__(self, dtype=None, copy=None):
        a = self.normalized()
        return a.astype(dtype) if dtype is not None else a


class CudaScorer:
    """Sub-patch mass of (ancestor) heat maps with the sm_90a kernels; one D2H of a few scalars per expansion."""

    def from_low_res(self, low_res, h, w):
        hm, stats = ops.heatmap(low_res.contiguous(), h, w, clamp=True, with_stats=True)
        return Heatmap(hm, stats, h, w)

    def from_full_res(self, tensor, h, w):
        """a vsm object that already returns the H x W map (generic VSM.inference API): upload if needed, then reduce"""
        t = tensor.reshape(h, w)
        if not t.is_cuda:
            t = t.cuda()
        t = t.float().contiguous()
        # identity resample (LH=h, LW=w) reuses the heat-map kernel for clamp + (max,min,sum)
        hm, stats = ops.heatmap(t, h, w, clamp=True, with_stats=True)
        return Heatmap(hm, stats, h, w)

    def rect_sums(self, jobs):
        """jobs: list of (Heatmap, rects int [n,4]); returns list of float64 arrays; a single sync."""
        outs = []
        for hmap, rects in jobs:
            r = torch.tensor(np.asarray(rects, dtype=np.int32), device=hmap.map.device)
            outs.append(ops.rect_sums(hmap.map, r, hmap.stats))
        cat = torch.cat(outs).cpu().numpy()
        res, o = [], 0
        for _, rects in jobs:
            res.append(cat[o:o + len(rects)])
            o += len(rects)
        return res


class MapPyramid:
    """rectangle sums of a node's normalised map computed on demand from a materialised Heatmap (generic vsm objects that
    return the H x W map, and the weak-cue branch whose map comes from a second inference)"""

    def __init__(self, scorer, heat, bbox):
        self.scorer, self.heat, self.bbox = scorer, heat, [int(v) for v in bbox]
        self.sums = {}

    @property
    def stats(self):
        return self.heat.host_stats()

    def missing(self, rects):
        return [r for r in rects if r not in self.sums]

    def relative(self, rects):
        return [[r[0] - self.bbox[0], r[1] - self.bbox[1], r[2], r[3]] for r in rects]

    def get(self, rect):
        return self.sums[rect]


def fill_pyramids(scorer, wanted):
    """wanted: list of (pyramid, rects).  All sums that are not in a record come from ONE scorer.rect_sums call (one sync)."""
    jobs = [(p, p.missing(rects)) for p, rects in wanted]
    jobs = [(p, m) for p, m in jobs if m]
    if not jobs:
        return
    res = scorer.rect_sums([(p.heat, p.relative(m)) for p, m in jobs])
    for (p, m), vals in zip(jobs, res):
        for r, v in zip(m, vals):
            p.sums[r] = v


class LazyHeat:
    """search_path[i]['final_heatmap'] without paying for it: the reference stores normalize_score(map) as a [h,w,1] fp32
    numpy array per expanded node (visual_search.py:448) although only the visualiser reads it; here the array is
    materialised from the node's low-res mask when somebody converts it (np.asarray)."""

    def __init__(self, scorer, low_res, h, w, fetch=None):
        self.scorer, self.low_res, self.h, self.w, self.fetch = scorer, low_res, h, w, fetch
        self._heat = None

    def heat(self):
        if self._heat is None:
            low = self.low_res if self.low_res is not None else (self.fetch() if self.fetch is not None else None)
            if low is None:
                raise RuntimeError("this node's low-res mask lives on another rank (sharded frontier) and was not fetched")
            self._heat = self.scorer.from_low_res(low, self.h, self.w)
        return self._heat

    def __array__(self, dtype=None, copy=None):
        a = np.asarray(self.heat())
        return a.astype(dtype) if dtype is not None else a


def _sub_scores_from_sums(sums, n_children):
    """get_subpatch_scores (visual_search.py:255-266) given rectangle sums of the normalised map: sums[:n] children,
    sums[n] whole patch.  Arithmetic in numpy float32 like the reference's `.sum()` results."""
    total = np.float32(sums[n_children])
    out = []
    for i in range(n_children):
        s = np.float32(sums[i])
        if total > 0:
            s = np.float32(s / total)
        else:
            s = np.float32(s * 0)
        out.append(s)
    return out


# ---------------------------------------------------------------------------------------------------------------
# one search as an explicit state machine
# ---------------------------------------------------------------------------------------------------------------
class _NodeEval:
    """Outputs of one detection-mode evaluation of a crop, reduced to what the controller consumes."""
    __slots__ = ("top_logit", "top_box", "n_logits", "boxes", "scores", "low_res", "full_map", "heat", "pyramid", "n_valid",
                 "valid_boxes", "fetch_valid", "fetch_low_res")

    def __init__(self):
        self.top_logit = None    # python float (sigmoid score)
        self.top_box = None      # torch CPU float32 [4] cxcywh in (0,1)
        self.n_logits = 0
        self.boxes = None        # full [P,4] (device; needed only when the record's 16 valid boxes overflow)
        self.scores = None
        self.low_res = None      # [4g,4g] fp32 device (None for crops evaluated by another rank)
        self.full_map = None     # H x W tensor from a generic vsm.inference
        self.heat = None         # Heatmap once materialised
        self.pyramid = None      # RecordPyramid (record path) - None for generic vsm objects
        self.n_valid = None      # rows with score > 0.5 (record path)
        self.valid_boxes = None  # torch CPU [min(n_valid,16), 4] cxcywh (record path)
        self.fetch_valid = None  # callable -> all valid boxes, for n_valid > 16 (owner rank's device copy / broadcast)
        self.fetch_low_res = None

    @classmethod
    def from_record(cls, row, bbox, smallest_size):
        r = parse_record(row, bbox, smallest_size)
        if r["top_index"] < 0 and r["n_logits"] > 0:
            raise RuntimeError("crop evaluation produced no finite detection score (NaN logits)")
        ev = cls()
        ev.top_logit, ev.n_logits, ev.n_valid = r["top_logit"], r["n_logits"], r["n_valid"]
        ev.top_box = torch.from_numpy(r["top_box"])
        ev.valid_boxes = torch.from_numpy(r["valid_boxes"])
        ev.pyramid = r["pyramid"]
        return ev


class SearchState:
    def __init__(self, image, target_object_name, smallest_size, confidence_high=0.5, confidence_low=0.3,
                 target_cue_threshold=6.0, target_cue_threshold_decay=0.7, target_cue_threshold_minimum=3.0):
        self.image = image
        self.target = target_object_name
        self.smallest_size = smallest_size
        self.confidence_high, self.confidence_low = confidence_high, confidence_low
        self.thr, self.thr_decay, self.thr_min = target_cue_threshold, target_cue_threshold_decay, target_cue_threshold_minimum
        init_patch = dict(bbox=[0, 0, image.width, image.height], scale_level=1, score=None, parent_index=-1)
        self.search_path = [init_patch]
        self.queue = PriorityQueue()
        self.current = init_patch
        self.cache = {}               # bbox tuple -> _NodeEval
        self.pending = set()          # bbox tuples whose evaluation is in flight
        self.gen = None               # commit of the current node in progress (generator, see SearchController._process)
        self.request = None           # ("vqa" | "segmentation", question) the commit is waiting for
        self.reply = None
        self.done = False
        self.success = False
        self.all_valid_boxes = None
        self.n_evals = 0

    # -- frontier ------------------------------------------------------------------------------------------
    @staticmethod
    def key(patch):
        return tuple(int(v) for v in patch["bbox"])

    def _free(self, patch):
        k = self.key(patch)
        return k not in self.cache and k not in self.pending

    def wanted(self, k):
        """Nodes whose evaluation is (or is likely to be) needed next and is neither cached nor in flight: the current node
        first, then the best queue entries (speculation; does not touch the heap order)."""
        out = []
        if self.done or k <= 0:
            return out
        if self._free(self.current):
            out.append(self.current)
        if k > len(out):
            for pr in sorted(self.queue.queue):
                if len(out) >= k:
                    break
                if self._free(pr.item) and all(pr.item is not o for o in out):
                    out.append(pr.item)
        return out

    def crop(self, patch):
        b = patch["bbox"]
        return self.image.crop((int(b[0]), int(b[1]), int(b[0] + b[2]), int(b[1] + b[3])))


class SearchController:
    """Runs one or many SearchStates against a vsm object, batching (and pipelining) node evaluations."""

    def __init__(self, vsm, scorer=None, batch_size=1, extract_noun_chunks=None, depth=2, split_min=8, speculate_children=True):
        self.vsm = vsm
        self.scorer = scorer if scorer is not None else CudaScorer()
        self.batch_size = max(1, int(batch_size))
        if extract_noun_chunks is None:
            # the reference always parses the location phrase with spaCy (visual_search.py:435); the default here does the
            # same and RAISES if spaCy is missing rather than silently using "region {phrase}" for every node
            from .noun_chunks import extract_noun_chunks as _enc
            extract_noun_chunks = _enc
        self.extract_noun_chunks = extract_noun_chunks
        self.regions = hasattr(vsm, "detect_regions")
        self.batched = self.regions or hasattr(vsm, "detect_batch")
        self.pipelined = hasattr(vsm, "detect_regions_launch")
        self.depth = max(1, int(depth))
        self.split_min = split_min
        self.speculate_children = speculate_children
        self.batches = []              # sizes of the launched batches (diagnostics)
        self.cue_batches = []          # (kind, size) of the batched weak-cue calls

    # -- evaluation ----------------------------------------------------------------------------------------
    def _launch(self, requests):
        """asynchronous: the GPU work of the batch is queued, nothing is waited for"""
        for st, p in requests:
            st.pending.add(st.key(p))
        questions = [DETECTION_QUESTION.format(st.target) for st, p in requests]
        handle = self.vsm.detect_regions_launch([(st.image, p["bbox"]) for st, p in requests], questions,
                                                [st.smallest_size for st, p in requests])
        self.batches.append(len(requests))
        return requests, handle

    def _collect(self, inflight):
        requests, handle = inflight
        results = self.vsm.detect_regions_finish(handle)
        for (st, p), ev in zip(requests, results):
            k = st.key(p)
            st.pending.discard(k)
            st.cache[k] = ev
            st.n_evals += 1

    def _evaluate(self, requests):
        """synchronous evaluation (vsm objects without the launch/finish API).  Fills state.cache."""
        if not requests:
            return
        self.batches.append(len(requests))
        if self.batched:
            questions = [DETECTION_QUESTION.format(st.target) for st, p in requests]
            if self.regions:       # the crop is cut on the GPU from the resident search image
                results = self.vsm.detect_regions([(st.image, p["bbox"]) for st, p in requests], questions)
            else:
                results = self.vsm.detect_batch([st.crop(p) for st, p in requests], questions)
            for (st, p), ev in zip(requests, results):
                st.cache[st.key(p)] = ev
                st.n_evals += 1
            return
        import copy
        for st, p in requests:
            patch_img = st.crop(p)
            boxes, logits, hm = self.vsm.inference(copy.deepcopy(patch_img), DETECTION_QUESTION.format(st.target), mode="detection")
            ev = _NodeEval()
            ev.n_logits = len(logits)
            if ev.n_logits > 0:
                flat = logits.view(-1)
                ti = int(flat.argmax())
                ev.top_logit = flat.max()
                ev.top_box = boxes[ti].view(4).clone()
                ev.boxes, ev.scores = boxes, logits
            ev.full_map = hm
            st.cache[st.key(p)] = ev
            st.n_evals += 1

    # -- one node, exactly visual_search_queue's body (visual_search.py:390-473) -----------------------------
    def _process(self, st: SearchState):
        """Generator: runs the node's commit logic and YIELDS ("vqa" | "segmentation", question) whenever the weak-cue branch
        needs another model call on the node's crop; the controller answers with the result (send) - batched over all the
        searches that are waiting at the same point (the reference does these calls inline, one node at a time,
        visual_search.py:427-443).  Returns True when the search ends successfully at this node."""
        cur = st.current
        bb = cur["bbox"]
        lvl = cur["scale_level"]
        ev = st.cache[st.key(cur)]
        pw, ph = int(bb[0] + bb[2]) - int(bb[0]), int(bb[1] + bb[3]) - int(bb[1])
        if ev.n_logits > 0:
            top_logit = ev.top_logit
            final_bbox = ev.top_box.view(4) * torch.Tensor([pw, ph, pw, ph])
            final_bbox[:2] -= final_bbox[2:] / 2
            if top_logit > st.confidence_high:
                st.search_path[-1]["detection_result"] = final_bbox
                if len(st.search_path) == 1:
                    st.all_valid_boxes = self._all_valid(ev, pw, ph)
                return True
            st.search_path[-1]["temp_detection_result"] = (top_logit, final_bbox)
        if min(bb[2], bb[3]) <= st.smallest_size:
            return False
        h, w = bb[3], bb[2]
        idx = len(st.search_path) - 1
        if ev.pyramid is not None:                 # record path: statistics and sums arrived with the batch
            pyr = ev.pyramid
            final_heat = LazyHeat(self.scorer, ev.low_res, h, w, ev.fetch_low_res)
        else:
            if ev.heat is None:
                ev.heat = self.scorer.from_low_res(ev.low_res, h, w) if ev.low_res is not None else self.scorer.from_full_res(ev.full_map, h, w)
            pyr = MapPyramid(self.scorer, ev.heat, bb)
            final_heat = ev.heat
        subs, _, _ = get_sub_patches(bb, *split_4subpatches(bb))
        sub_keys = [tuple(int(v) for v in s) for s in subs]

        def chain(pyr_of_cur):
            out = []
            tmp = cur
            while True:
                out.append((pyr_of_cur if tmp is cur else tmp["_pyr"], sub_keys + [tuple(int(v) for v in tmp["bbox"])], tmp["scale_level"]))
                if tmp["parent_index"] == -1:
                    break
                tmp = st.search_path[tmp["parent_index"]]
            return out

        # optimistic strong-cue path: whatever is not already in a record comes back in ONE device->host copy
        terms = chain(pyr)
        fill_pyramids(self.scorer, [(t[0], t[1]) for t in terms])
        score_max = float(pyr.stats[0])
        threshold = max(st.thr_min, st.thr * (st.thr_decay) ** (lvl - 1))
        if not (score_max > threshold):
            # weak cue: ask the VSM where the object would be, then segment that region (visual_search.py:427-443)
            vqa_results = yield ("vqa", CUE_QUESTION.format(st.target))
            phrase = vqa_results.split("most likely to appear")[-1].strip()
            if phrase.endswith("."):
                phrase = phrase[:-1]
            phrase = phrase.split(st.target)[-1]
            chunks = self.extract_noun_chunks(phrase)
            phrase = chunks[0] if len(chunks) == 1 else "region {}".format(phrase)
            cue = yield ("segmentation", DETECTION_QUESTION.format(phrase))
            st.search_path[idx]["context_cue"] = vqa_results + "#" + phrase
            if isinstance(cue, _NodeEval) and cue.pyramid is not None:      # cue map as a crop record (statistics + quad-tree sums)
                pyr = cue.pyramid
                final_heat = LazyHeat(self.scorer, cue.low_res, h, w, cue.fetch_low_res)
            else:
                final_heat = cue if isinstance(cue, Heatmap) else self.scorer.from_full_res(cue, h, w)
                pyr = MapPyramid(self.scorer, final_heat, bb)
            terms = chain(pyr)
            fill_pyramids(self.scorer, [(t[0], t[1]) for t in terms])
        st.search_path[idx]["_pyr"] = pyr
        st.search_path[idx]["final_heatmap"] = final_heat      # lazily converts to the reference's [h,w,1] numpy array
        basic = [0] * len(subs)
        for p_t, keys, level in terms:
            tmp_scores = _sub_scores_from_sums([p_t.get(k) for k in keys], len(subs))
            basic = [basic[i] + tmp_scores[i] / (4 ** level) for i in range(len(subs))]
        for sp, sc in zip(subs, basic):
            info = dict(bbox=sp, scale_level=lvl + 1, score=sc, parent_index=idx)
            st.queue.put(Prioritize(-info["score"], info))
        return False

    @staticmethod
    def _all_valid(ev, pw, ph):
        # visual_search.py:406-410 (only when the root itself succeeds)
        if ev.valid_boxes is not None and ev.n_valid is not None:
            av = ev.valid_boxes if ev.n_valid <= ev.valid_boxes.shape[0] else ev.fetch_valid()
            av = av.clone().view(-1, 4)
        else:
            boxes, scores = ev.boxes, ev.scores
            if boxes.is_cuda:
                boxes, scores = boxes.cpu(), scores.cpu()
            av = boxes[scores.view(-1) > 0.5].view(-1, 4)
        av = av * torch.Tensor([[pw, ph, pw, ph]])
        av[:, :2] -= av[:, 2:] / 2
        return av

    def _advance(self, st: SearchState):
        """Commit as many nodes as the cache allows, in the reference's pop order.  Stops when the current node has not been
        evaluated yet, or when its commit is waiting for a weak-cue model call (st.request is then set)."""
        while not st.done:
            if st.gen is None:
                if st.key(st.current) not in st.cache:
                    return
                st.gen = self._process(st)
                reply = None
            else:
                if st.request is not None:
                    return                                  # still waiting for _serve_cues
                reply, st.reply = st.reply, None
            try:
                st.request = st.gen.send(reply)
                return                                      # parked: a weak-cue call is pending
            except StopIteration as fin:
                ok = bool(fin.value)
            st.gen = None
            if ok:
                st.done, st.success = True, True
                return
            if st.queue.empty():
                st.done = True
                return
            st.current = st.queue.get().item
            st.search_path.append(st.current)

    def _serve_cues(self, states):
        """answer the pending weak-cue calls of all parked searches: one batched model call per kind when the vsm offers
        `inference_many`, the reference's one-crop-at-a-time `inference` otherwise"""
        parked = [st for st in states if st.request is not None and not st.done]
        if not parked:
            return False
        for kind in ("vqa", "segmentation"):
            group = [st for st in parked if st.request is not None and st.request[0] == kind]
            if not group:
                continue
            if hasattr(self.vsm, "inference_many"):
                extra = {}
                if kind == "segmentation" and getattr(self.vsm, "cue_records", False):
                    extra["smallest_sizes"] = [st.smallest_size for st in group]      # -> cue maps come back as crop records
                replies = self.vsm.inference_many([(st.image, st.current["bbox"]) for st in group], [st.request[1] for st in group], kind,
                                                  **extra)
            else:
                import copy
                replies = [self.vsm.inference(copy.deepcopy(st.crop(st.current)), st.request[1], mode=kind) for st in group]
            for st, r in zip(group, replies):
                st.reply, st.request = r, None
            self.cue_batches.append((kind, len(group)))
        return True

    def _select(self, active, limit):
        """mandatory nodes first (the current node of every search that is not already in flight), then fill the batch with
        speculation, round-robin over the active searches: the best queue entries, and - if the batch still has room - the
        CHILDREN of the nodes being evaluated (their geometry is known before the parent commits, visual_search.py:234-253), so
        that a search whose frontier is one node deep does not pay one GPU round per tree level"""
        reqs = [(st, st.current) for st in active if st._free(st.current)][:limit]
        room = limit - len(reqs)
        if room > 0 and active:
            per = max(1, room // len(active)) + 1
            extra = []
            for st in active:
                taken = [p for s2, p in reqs if s2 is st]
                for p in st.wanted(per + len(taken)):
                    if all(p is not t for t in taken):
                        extra.append((st, p))
            reqs += extra[:room]
            room = limit - len(reqs)
        if room > 0 and self.speculate_children:
            seen = {(id(st), st.key(p)) for st, p in reqs}
            kids = []
            for st, p in list(reqs):
                bb = p["bbox"]
                if not expandable(bb, st.smallest_size):
                    continue
                subs, _, _ = get_sub_patches(bb, *split_4subpatches(bb))
                for sp in subs:
                    node = dict(bbox=sp, scale_level=p["scale_level"] + 1, score=None, parent_index=None)     # evaluation only
                    if st._free(node) and (id(st), st.key(node)) not in seen:
                        seen.add((id(st), st.key(node)))
                        kids.append((st, node))
            reqs += kids[:room]
        return reqs

    def run(self, states):
        """run a fixed list of searches together until the last one ends; results in the order of `states`"""
        results = {id(st): res for st, res in self.stream(states)}
        return [results[id(st)] for st in states]

    def stream(self, states, window=None):
        """Continuous admission: take searches from the iterable `states` as they are needed, keep at most `window` of them
        active (None = all at once), and yield (state, result) for each search as soon as it ends.  A finished search frees its
        slot for the next one before the next frontier batch is selected, so batches mix searches at different depths.  The
        controller holds no reference to a yielded state; speculative crops of it that are still in flight are dropped with
        their batch.  Sets `t_admit` / `t_done` (time.perf_counter) on every state."""
        import time
        from collections import deque
        feed = iter(states)
        more = True
        active = []
        inflight = deque()
        while True:
            for st in active:
                self._advance(st)
            if any(st.done for st in active):
                finished = [st for st in active if st.done]
                active = [st for st in active if not st.done]
                for st in finished:
                    st.t_done = time.perf_counter()
                    yield st, self._finish(st)
                del finished, st
            while more and (window is None or len(active) < window):
                st = next(feed, None)
                if st is None:
                    more = False
                    break
                st.t_admit = time.perf_counter()
                active.append(st)
            if self._serve_cues(active):
                continue               # replies are in: let the parked commits run on before evaluating more crops
            if not active:
                break                  # speculative batches still in flight are simply dropped
            if not self.pipelined:
                self._evaluate(self._select(active, self.batch_size))
                continue
            while len(inflight) < self.depth:
                reqs = self._select(active, self.batch_size)
                if not reqs:
                    break
                if not inflight and self.depth > 1 and len(reqs) >= 2 * self.split_min:
                    # nothing queued behind this batch: cut it in two so that the second half runs on the GPU while the host
                    # commits the first half and launches its successors
                    half = (len(reqs) + 1) // 2
                    inflight.append(self._launch(reqs[:half]))
                    inflight.append(self._launch(reqs[half:]))
                else:
                    inflight.append(self._launch(reqs))
            if not inflight:
                raise RuntimeError("search controller stalled: active searches but nothing to evaluate")
            self._collect(inflight.popleft())

    @staticmethod
    def _finish(st: SearchState):
        # visual_search.py:496-516
        path_length = len(st.search_path)
        final_step = st.search_path[-1]
        ok = st.success
        if not ok:
            max_logit, final_step, path_length = 0, None, 0
            for i, step in enumerate(st.search_path):
                if "temp_detection_result" in step and step["temp_detection_result"][0] > max_logit:
                    max_logit, final_step, path_length = step["temp_detection_result"][0], step, i + 1
            if final_step is None:
                raise RuntimeError("no detection result on any search step (the reference dereferences None here: "
                                   "visual_search.py:509)")
            final_step["detection_result"] = final_step["temp_detection_result"][1]
            if max_logit >= st.confidence_low:
                ok = True
        return final_step, path_length, ok, st.all_valid_boxes


def visual_search(vsm, image, target_object_name, target_bbox, smallest_size, confidence_high=0.5, confidence_low=0.3,
                  target_cue_threshold=6.0, target_cue_threshold_decay=0.7, target_cue_threshold_minimum=3.0,
                  visualize=False, save_path=None, scorer=None, batch_size=None, extract_noun_chunks=None,
                  return_state=False, depth=2):
    """Same contract as the reference's visual_search() (visual_search.py:484-516)."""
    if visualize:
        assert save_path is not None
    st = SearchState(image, target_object_name, smallest_size, confidence_high, confidence_low, target_cue_threshold,
                     target_cue_threshold_decay, target_cue_threshold_minimum)
    if batch_size is None:
        batch_size = getattr(vsm, "frontier_batch", 1)
    ctl = SearchController(vsm, scorer, batch_size, extract_noun_chunks, depth=depth)
    res = ctl.run([st])[0]
    if visualize:                          # visual_search.py:512-514
        from .visualize import visualize_search_path
        vis_len = res[1] if res[2] else len(st.search_path)
        visualize_search_path(image, st.search_path, vis_len, target_bbox, target_object_name, save_path)
    return res + (st,) if return_state else res


def visual_search_many(vsm, jobs, batch_size=8, scorer=None, extract_noun_chunks=None, depth=2, **kw):
    """Run several independent searches in lock-step so their frontiers share GPU batches.
    jobs: list of (image, target_object_name, smallest_size).  depth: frontier batches in flight.  Returns (results, states)."""
    states = [SearchState(img, name, ss, **kw) for img, name, ss in jobs]
    ctl = SearchController(vsm, scorer, batch_size, extract_noun_chunks, depth=depth)
    return ctl.run(states), states


# ---------------------------------------------------------------------------------------------------------------
# search-only V*Bench evaluation (visual_search.py:520-564)
# ---------------------------------------------------------------------------------------------------------------
def _decode(path):
    from PIL import Image
    with Image.open(path) as im:
        return im.convert("RGB")


def _benchmark_images(args, pool, lookahead):
    """(test_type, image_file, [(gt_bbox, target_object)], PIL image) per image with at least one target, in the reference's
    order: direct_attributes then relative_position, files in os.listdir order.  Images are decoded on `pool`, `lookahead`
    images ahead of the caller.  The annotation is the image FILE name cut at its first '.' (bench_eval.list_samples); the
    reference cuts the whole path there, which breaks under a directory whose name contains a dot."""
    from collections import deque
    from .bench_eval import TEST_TYPES, list_samples

    def entries():
        for test_type in TEST_TYPES:
            if args.visualization:
                os.makedirs(os.path.join(args.output_path, test_type), exist_ok=True)
            for image_file, image_path, annotation_path in list_samples(os.path.join(args.benchmark_folder, test_type)):
                with open(annotation_path) as f:
                    ann = json.load(f)
                targets = list(zip(ann["bbox"], ann["target_object"]))
                if targets:
                    yield test_type, image_file, targets, image_path

    ahead = deque()
    for entry in entries():
        ahead.append((entry, pool.submit(_decode, entry[3])))
        if len(ahead) > lookahead:
            (test_type, image_file, targets, _), fut = ahead.popleft()
            yield test_type, image_file, targets, fut.result()
    while ahead:
        (test_type, image_file, targets, _), fut = ahead.popleft()
        yield test_type, image_file, targets, fut.result()


def main(args, vsm=None, scorer=None, extract_noun_chunks=None):
    """The reference's search-only benchmark: one visual_search() per annotated target of V*Bench, then the two lines it prints
    (average search path length over the hits, Top-1 accuracy at IoU > 0.5).  Same arguments, thresholds, per-target logic
    and visualisation files.  The schedule differs: up to --searches-in-flight searches run at once in one SearchController,
    the next target is admitted as soon as one ends, and the frontier batches mix their crops.  Every search is
    independent of the others, so the per-target results do not depend on the window.  `vsm` may be injected; otherwise it
    is built from the arguments as the reference does.  Returns the per-target records (see --trajectory-json)."""
    from concurrent.futures import ThreadPoolExecutor
    from .seal import smallest_size_for
    args = parse_args(args)
    if vsm is None:
        from .vsm import VSM
        vsm = VSM(args)
    window = max(1, int(args.searches_in_flight))
    ctl = SearchController(vsm, scorer, args.search_batch, extract_noun_chunks)
    release = getattr(vsm, "release", None)
    held = {}                  # id(image) -> [image, targets not finished yet]
    thresholds = dict(confidence_high=args.confidence_high, confidence_low=args.confidence_low,
                      target_cue_threshold=args.target_cue_threshold, target_cue_threshold_decay=args.target_cue_threshold_decay,
                      target_cue_threshold_minimum=args.target_cue_threshold_minimum)

    def states(images):
        n = 0
        for test_type, image_file, targets, image in images:
            smallest = smallest_size_for(image, args.minimum_size_scale, args.minimum_size)
            held[id(image)] = [image, len(targets)]
            for i, (gt_bbox, object_name) in enumerate(targets):
                st = SearchState(image, object_name, smallest, **thresholds)
                st.sample = dict(order=n, test_type=test_type, image=image_file, target_index=i, target=object_name, gt_bbox=gt_bbox)
                n += 1
                yield st

    records = []
    with ThreadPoolExecutor(max_workers=1) as pool:
        feed = states(_benchmark_images(args, pool, lookahead=max(2, window)))
        for st, (final_step, path_length, ok, _) in ctl.stream(feed, window):
            smp = st.sample
            if args.visualization:           # visual_search.py:512-514, before main shifts the box (:552-555)
                from .visualize import visualize_search_path
                vis_path = os.path.join(args.output_path, smp["test_type"], "{}_{}".format(smp["image"].split(".")[0], smp["target_index"]))
                visualize_search_path(st.image, st.search_path, path_length if ok else len(st.search_path), smp["gt_bbox"],
                                      smp["target"], vis_path)
            box, patch = final_step["detection_result"], final_step["bbox"]
            if ok:
                box[0] += patch[0]           # in place, as the reference does
                box[1] += patch[1]
            else:
                box = box.clone()
                box[0] += patch[0]
                box[1] += patch[1]
            iou_i = float(iou(box, smp["gt_bbox"]))
            smp.update(search_successful=bool(ok), path_length=int(path_length), final_box=[float(v) for v in box], iou=iou_i,
                       accuracy=(1.0 if iou_i > 0.5 else 0.0) if ok else 0,
                       expanded=[dict(bbox=[int(v) for v in node["bbox"]], score=None if node["score"] is None else float(node["score"]),
                                      context_cue=node.get("context_cue")) for node in st.search_path],
                       evaluations=st.n_evals, latency_s=st.t_done - st.t_admit)
            records.append(smp)
            entry = held[id(st.image)]
            entry[1] -= 1
            if entry[1] == 0:                # last target of the image: drop its resident device copy now
                del held[id(st.image)]
                if release is not None:
                    release(st.image)
    records.sort(key=lambda r: r.pop("order"))
    acc_list = [r["accuracy"] for r in records]
    search_path_length_list = [r["path_length"] if r["search_successful"] else 0 for r in records]
    avg_len = np.mean([search_path_length_list[i] for i in range(len(search_path_length_list)) if acc_list[i]])
    top1 = np.mean(acc_list)
    print("Avg search path length:", avg_len)
    print("Top 1 Acc:", top1)
    if args.trajectory_json:
        def num(x):
            return None if np.isnan(x) else float(x)
        with open(args.trajectory_json, "w") as f:
            json.dump(dict(avg_search_path_length=num(avg_len), top1_acc=num(top1), searches_in_flight=window,
                           search_batch=args.search_batch, samples=records), f, indent=1)
    return records


if __name__ == "__main__":
    # run the package's copy of this module: vsm.py imports it, and the controller's isinstance checks need ONE set of classes
    from vstar_b200.visual_search import main as _main
    _main(sys.argv[1:])
