"""Test-only helpers (NOT product code): a numpy heat-map scorer so the search controller's ordering logic can be
checked on a CPU-only box, and the deterministic stub VSM used by the committed search goldens."""
import os
import tempfile

import numpy as np
import torch


class NumpyHeat:
    def __init__(self, arr):
        self.arr = arr                       # clamped [h,w] fp32
        self.h, self.w = arr.shape

    def host_stats(self):
        return np.array([self.arr.max(), self.arr.min(), self.arr.sum()], np.float32)

    def norm(self):
        if getattr(self, "_n", None) is None:
            mx, mn = self.arr.max(), self.arr.min()
            self._n = ((self.arr - mn) / (mx - mn) if mx != mn else self.arr * 0).astype(np.float64)
        return self._n

    def __array__(self, dtype=None, copy=None):
        # what the reference stores in search_path[i]['final_heatmap']: normalize_score in fp32, [h,w,1] (visual_search.py:268-275, :448)
        mx, mn = self.arr.max(), self.arr.min()
        a = ((self.arr - mn) / (mx - mn) if mx != mn else self.arr * 0).astype(np.float32).reshape(self.h, self.w, 1)
        return a.astype(dtype) if dtype is not None else a


class NumpyScorer:
    """restates ops.heatmap / ops.rect_sums with numpy (float64 sums of the normalised map)"""

    def from_low_res(self, low_res, h, w):
        t = torch.nn.functional.interpolate(low_res.float().cpu()[None, None], (h, w), mode="bilinear", align_corners=False)[0, 0]
        return NumpyHeat(t.clamp(min=0).numpy())

    def from_full_res(self, tensor, h, w):
        return NumpyHeat(tensor.reshape(h, w).float().cpu().clamp(min=0).numpy())

    def rect_sums(self, jobs):
        out = []
        for heat, rects in jobs:
            n = heat.norm()
            out.append(np.array([n[max(0, y):y + rh, max(0, x):x + rw].sum() for x, y, rw, rh in rects]))
        return out


VQA_ANSWERS = (
    "The object is most likely to appear near the table.",
    "The mug is most likely to appear on the wooden shelf near the window.",
    "It is most likely to appear in the upper left.",
    "The mug is most likely to appear beside the red kettle.",
    "It is most likely to appear somewhere high.",
    "The mug is most likely to appear near the sink, the lamp.",
)


class StubVSM:
    # pure function of (crop pixels, question).  hot: None = detection logits stay below 0.45 (never confident); "root" = crops
    # with min side >= 600 get three confident boxes (0.9 / 0.7 / 0.6); "small" = crops with min side <= 300 get one confident
    # box (0.8).  The 'vqa' answer is one of VQA_ANSWERS picked by the crop; the 'segmentation' map depends on the QUESTION too,
    # so the context-cue phrase (noun-chunk logic, visual_search.py:430-442) changes the trajectory.
    def __init__(self, hot=None):
        self.calls = []
        self.hot = hot

    def _eval(self, image, question, mode):
        """-> (answer str | None, boxes, logits, low [12,12]) - pure function of (crop pixels, question, mode)"""
        import zlib
        arr = np.asarray(image, dtype=np.uint8)
        h, w = arr.shape[:2]
        self.calls.append((w, h, {"detection": 0, "vqa": 1, "segmentation": 2}[mode]))
        s = int(arr[::max(1, h // 16), ::max(1, w // 16)].astype(np.int64).sum()) % (2 ** 31)
        if mode == "vqa":
            return VQA_ANSWERS[s % len(VQA_ANSWERS)], None, None, None
        if mode == "segmentation":
            s = (s ^ zlib.crc32(question.encode())) % (2 ** 31)
        rng = np.random.default_rng(s)
        low = rng.standard_normal((12, 12)).astype(np.float32) * 4.0
        if mode == "segmentation":
            return None, None, None, low
        logits = torch.from_numpy(rng.uniform(0.0, 0.45, (2304, 1)).astype(np.float32))
        boxes = torch.from_numpy(rng.uniform(0.1, 0.9, (2304, 4)).astype(np.float32))
        if self.hot == "root" and min(w, h) >= 600:
            logits[100, 0], logits[7, 0], logits[2000, 0] = 0.9, 0.7, 0.6
        if self.hot == "small" and min(w, h) <= 300:
            logits[55, 0] = 0.8
        if self.hot == "many" and min(w, h) >= 600:
            logits[40:70, 0] = torch.linspace(0.95, 0.55, 30)           # 30 boxes above 0.5: more than a record's 16 slots
        return None, boxes, logits, low

    def inference(self, image, question, mode="segmentation"):
        ans, boxes, logits, low = self._eval(image, question, mode)
        if mode == "vqa":
            return ans
        h, w = image.height, image.width
        hm = torch.nn.functional.interpolate(torch.from_numpy(low)[None, None], (h, w), mode="bilinear",
                                             align_corners=False)[0, 0].clamp(min=0)
        if mode == "segmentation":
            return hm
        return boxes, logits, hm


def pack_record_numpy(boxes, logits, low, bbox, smallest, R):
    """TEST-side restatement of the crop-record layout (vstar_b200/records.py, csrc/heads.cu) with numpy; logits None = the
    record of a cue segmentation (heat-map part only)"""
    from vstar_b200 import records as RC
    row = np.zeros(R, np.float32)
    if logits is not None:
        sc = logits.view(-1).numpy()
        ti = int(sc.argmax())
        row[RC.REC_TOP], row[RC.REC_BOX:RC.REC_BOX + 4] = sc[ti], boxes[ti].numpy()
        row[RC.REC_NROWS], row[RC.REC_TOPIDX] = len(sc), ti
        valid = np.nonzero(sc > 0.5)[0]
        row[RC.REC_NVALID] = len(valid)
        for k, vi in enumerate(valid[:RC.REC_MAXVALID]):
            row[RC.REC_VALID + 4 * k:RC.REC_VALID + 4 * k + 4] = boxes[vi].numpy()
    rects = RC.pyramid_rects(bbox, smallest)
    if rects:
        heat = NumpyScorer().from_low_res(torch.from_numpy(low), int(bbox[3]), int(bbox[2]))
        row[RC.REC_MAX:RC.REC_MAX + 3] = heat.host_stats()
        row[RC.REC_NRECT] = len(rects)
        n = heat.norm()
        x0, y0 = int(bbox[0]), int(bbox[1])
        row[RC.REC_PYR:RC.REC_PYR + len(rects)] = [n[r[1] - y0:r[1] - y0 + r[3], r[0] - x0:r[0] - x0 + r[2]].sum() for r in rects]
    return row


class RecordStub(StubVSM):
    """the same pure function through the launch / finish RECORD interface the CUDA VSM exposes (CPU tensors here)"""

    def __init__(self, hot=None):
        super().__init__(hot)
        self.n_local = 0
        self.batches = []

    cue_records = True

    def detect_regions_launch(self, regions, questions, smallest_sizes, rec_len=None, mode="detection"):
        from vstar_b200 import records as RC
        R = max(rec_len or 0, RC.record_floats(max(len(RC.pyramid_rects(b, ss)) for (_, b), ss in zip(regions, smallest_sizes))))
        rec = torch.zeros((len(regions), R), dtype=torch.float32)
        keep = []
        self.batches.append(len(regions))
        for k, ((src, b), q, ss) in enumerate(zip(regions, questions, smallest_sizes)):
            self.n_local += 1
            im = src.crop((int(b[0]), int(b[1]), int(b[0] + b[2]), int(b[1] + b[3])))
            _, boxes, logits, low = self._eval(im, q, mode)
            rec[k] = torch.from_numpy(pack_record_numpy(boxes, logits, low, b, ss, R))
            keep.append((boxes, logits, torch.from_numpy(low)))
        return dict(rec=rec, keep=keep, regions=regions, smallest=list(smallest_sizes))

    def detect_regions_finish(self, h):
        from vstar_b200.visual_search import _NodeEval
        out = []
        for k, (boxes, logits, low) in enumerate(h["keep"]):
            ev = _NodeEval.from_record(h["rec"][k].numpy(), h["regions"][k][1], h["smallest"][k])
            ev.low_res, ev.boxes, ev.scores = low, boxes, logits
            if logits is not None:
                ev.fetch_valid = (lambda b=boxes, s=logits: b[s.view(-1) > 0.5].view(-1, 4))
            out.append(ev)
        return out

    def detect_regions(self, regions, questions, smallest_sizes=None):
        if smallest_sizes is None:
            smallest_sizes = [max(1, min(int(b[2]), int(b[3])) // 2) for _, b in regions]
        return self.detect_regions_finish(self.detect_regions_launch(regions, questions, smallest_sizes))

    def inference_many(self, regions, questions, mode, smallest_sizes=None):
        self.cue_batches = getattr(self, "cue_batches", []) + [(mode, len(regions))]
        if mode == "segmentation" and smallest_sizes is not None:         # cue maps as crop records, like the CUDA VSM
            return self.detect_regions_finish(self.detect_regions_launch(regions, questions, smallest_sizes, mode="segmentation"))
        return [self.inference(src.crop((int(b[0]), int(b[1]), int(b[0] + b[2]), int(b[1] + b[3]))), q, mode) for (src, b), q in zip(regions, questions)]


# ---------------------------------------------------------------- deterministic stand-in for spaCy (noun-chunk tests / goldens)
class _Tok:
    def __init__(self, i, text):
        self.i, self.text = i, text
        self.pos_, self.dep_, self.head = "X", "dep", None
        self.children = []


class _Span:
    def __init__(self, toks):
        self.text = " ".join(t.text for t in toks)


class _Doc:
    def __init__(self, toks):
        self.toks = toks

    def __iter__(self):
        return iter(self.toks)

    def __len__(self):
        return len(self.toks)

    def __getitem__(self, k):
        return _Span(self.toks[k]) if isinstance(k, slice) else self.toks[k]


class FakeNLP:
    """Rule parser with spaCy's Token surface (.i .pos_ .dep_ .children, doc[a:b].text): whitespace tokens; lexicon POS tags;
    DET / ADJ / noun-before-noun attach to the next noun (det / amod / compound), a preposition attaches to the previous noun
    (prep) and takes the next noun as pobj, a relative clause marker ("that"/"which") hangs the rest under the previous noun
    (relcl).  Not linguistics - just a deterministic tree generator that exercises every branch of the chunk logic."""
    NOUNS = {"table", "shelf", "window", "kettle", "left", "corner", "room", "desk", "wall", "door", "cup", "mug", "counter",
             "kitchen", "side", "floor", "chair", "sink", "lamp", "bed", "street", "tree", "car", "sign", "sky"}
    PRONS = {"it", "them", "something"}
    ADJS = {"wooden", "red", "upper", "lower", "big", "small", "blue", "left-hand", "kitchen's", "old", "white"}
    DETS = {"the", "a", "an", "this"}
    PREPS = {"near", "on", "in", "beside", "of", "at", "under", "behind", "above", "next", "to", "by"}
    RELS = {"that", "which"}
    POSS = {"kitchen's", "room's"}

    def __call__(self, text):
        toks = [_Tok(i, w) for i, w in enumerate(text.split())]
        key = [t.text.lower().strip(".,;") for t in toks]
        for t, k in zip(toks, key):
            t.pos_ = ("NOUN" if k in self.NOUNS else "PRON" if k in self.PRONS else "ADJ" if k in self.ADJS else "DET" if k in self.DETS
                      else "ADP" if k in self.PREPS else "SCONJ" if k in self.RELS else "X")

        def attach(child, head, dep):
            if child.head is None and child is not head:
                child.head, child.dep_ = head, dep
                head.children.append(child)

        nouns = [t for t in toks if t.pos_ in ("NOUN", "PRON")]
        for n in nouns:                                   # left modifiers: contiguous DET/ADJ/NOUN run before the head
            j = n.i - 1
            while j >= 0 and toks[j].pos_ in ("ADJ", "DET", "NOUN") and toks[j].head is None:
                k = key[j]
                attach(toks[j], n, "poss" if k in self.POSS else "amod" if toks[j].pos_ == "ADJ" else "det" if toks[j].pos_ == "DET" else "compound")
                j -= 1
        for t in toks:                                    # prepositions / relative markers
            if t.pos_ in ("ADP", "SCONJ") and t.head is None:
                prev = [n for n in nouns if n.i < t.i and n.head is None or (n.i < t.i and n.dep_ == "pobj")]
                nxt = [n for n in nouns if n.i > t.i and n.head is None]
                if prev:
                    attach(t, prev[-1], "prep" if t.pos_ == "ADP" else "relcl")
                if nxt:
                    attach(nxt[0], t, "pobj")
        for t in toks:
            t.children.sort(key=lambda c: c.i)
        return _Doc(toks)


def synth_image(seed, w, h):
    from PIL import Image
    return Image.fromarray(np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8), "RGB")


# ---------------------------------------------------------------- V*Bench driver fixtures (tests/test_bench_eval.py)
MISSING_MSG = ("Sorry, I can not answer the question. Some visual information about the following objects is missing or "
               "unclear:")


class _Proc:
    image_mean = [0.48145466, 0.4578275, 0.40821073]


class StubVQA:
    """Deterministic stand-in for VQA_LLM (vstar_bench_eval.py:49-165): answers are pure functions of their arguments, so the
    option an implementation picks checks every string / box it fed in (focus message, normalised boxes, long/short flags)."""
    image_processor = _Proc()

    def __init__(self):
        self.log = []

    def free_form_inference(self, image, question, max_new_tokens=512):
        import zlib
        k = zlib.crc32(question.encode()) % 3
        self.log.append(("free", image.size, question))
        if k == 0:
            return "It is blue."
        if k == 1:
            return MISSING_MSG + " the red mug."
        return MISSING_MSG + " a dog, the blue umbrella, traffic light."

    def get_object_crop(self, image, bbox, patch_scale=1.0):
        return torch.tensor([round(float(v), 2) for v in bbox] + [patch_scale], dtype=torch.float32)

    def multiple_choices_inference(self, image, question, options, object_crops=None, images_long=None, objects_long=None):
        import zlib
        key = repr((image.size, question, options, None if object_crops is None else object_crops.round().tolist(),
                    images_long, objects_long))
        self.log.append(("choice", key))
        return zlib.crc32(key.encode()) % len(options)


# parity reports the GPU tests leave behind (informational; outside the source tree unless VSB_REPORT_DIR says otherwise)
REPORT_DIR = os.environ.get("VSB_REPORT_DIR") or os.path.join(tempfile.gettempdir(), "vsb_reports")


def make_bench_folder(root):
    """tiny synthetic V*Bench tree: <root>/{direct_attributes,relative_position}/{name}.jpg|.png + {name}.json"""
    import json
    import os
    spec = {"direct_attributes": [("sa_1", 31, 640, 400), ("sa_2", 32, 300, 520), ("sa_3", 33, 512, 512), ("sa_4", 34, 700, 260)],
            "relative_position": [("sa_5", 35, 480, 360), ("sa_6", 36, 256, 600), ("sa_7", 37, 900, 300)]}
    for test_type, items in spec.items():
        d = os.path.join(root, test_type)
        os.makedirs(d, exist_ok=True)
        for name, seed, w, h in items:
            synth_image(seed, w, h).save(os.path.join(d, name + ".png"))
            with open(os.path.join(d, name + ".json"), "w") as f:
                json.dump({"question": f"What is the colour of item {seed}?", "options": ["red", "blue", "green", "white"][:2 + seed % 3]}, f)
    return root
