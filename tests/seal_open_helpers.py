"""Test-only fixtures for open-ended SEAL answering (`vstar_b200.seal.answer_open`, the reference demo's inference(),
app.py:130-233): a character tokenizer, the scripted model answers and search outcomes of six cases, and a compact record of
the pixel tensors handed to the model.  tests/golden/seal_open_golden.json is the reference's own inference() run on these
cases (tools/make_seal_open_golden.py); tests/test_seal_open.py runs vstar_b200.seal on the same ones."""
import hashlib
import zlib

import numpy as np
import torch

from tests.helpers import MISSING_MSG, synth_image

FOCUS_MSG = "Additional visual information to focus on: "

# (question, image seed, width, height, direct answer, searches: object -> found).  Questions pass app.py's input check
# (letters, spaces and , . ! ? ' " only).
CASES = [
    ("What is it", 40, 300, 220, "It is a cat.", {}),
    ("What colour is the mug", 41, 260, 330, MISSING_MSG + " the red mug.", {"the red mug": True}),
    ("Where is the dog", 42, 340, 255, MISSING_MSG + " a dog, the umbrella.", {"a dog": True, "the umbrella": True}),
    ("Which letters are there", 43, 280, 280, MISSING_MSG + " a, b, c.", {"a": True, "b": True, "c": True}),
    ("Where is the key", 44, 230, 310, MISSING_MSG + " the key.", {"the key": False}),
    ("What is on the table", 45, 360, 240, MISSING_MSG + " a cup, the key, a hat.", {"a cup": True, "the key": False, "a hat": True}),
]


def case_image(case):
    _, seed, w, h, _, _ = case
    return synth_image(seed, w, h)


class CharTokenizer:
    """one id per character (ord + 3); 0 = unk, 1 = bos, 2 = eos.  Enough of the HF tokenizer surface for the prompt builders
    (tokenizer(text).input_ids with a leading bos, bos_token_id) and for batch_decode(..., skip_special_tokens=True)."""
    bos_token_id, eos_token_id = 1, 2

    class _Enc:
        def __init__(self, ids):
            self.input_ids = ids

    def __call__(self, text):
        return self._Enc([self.bos_token_id] + [ord(c) + 3 for c in text])

    def decode(self, ids, skip_special_tokens=True):
        return "".join(chr(int(i) - 3) for i in ids if int(i) >= 3)

    def batch_decode(self, seqs, skip_special_tokens=True):
        return [self.decode(list(s), skip_special_tokens) for s in seqs]


def answer_ids(prompt_ids):
    """the scripted model: new token ids (ending in eos) for a prompt.  A direct question gets its case's direct answer; a
    prompt with the focus message gets "final <crc of the prompt text>"."""
    tok = CharTokenizer()
    text = tok.decode(prompt_ids)
    if FOCUS_MSG in text:
        ans = "final answer {}".format(zlib.crc32(text.encode()) % 100000)
    else:
        ans = next(c[4] for c in CASES if text.endswith("\n" + c[0] + " ASSISTANT:"))
    return tok(ans).input_ids[1:] + [tok.eos_token_id]


def fake_search(name, image):
    """visual_search's (final_step, path_length, search_successful, all_valid_boxes) for the scripted outcome of `name`:
    a found object "a" has two instances (all_valid_boxes), other found objects one; a failed search keeps its box"""
    ok = next(s[name] for c in CASES for s in [c[5]] if name in s)
    k = zlib.crc32(name.encode())
    patch = [k % 50, k % 37, image.width // 2, image.height // 2]
    box = torch.tensor([5.0 + k % 7, 9.0 + k % 5, 20.0 + k % 11, 30.0 + k % 3])
    valid = [box.clone(), box + 1] if ok and name == "a" else None
    return dict(bbox=patch, detection_result=box.clone()), 2, ok, valid


_IDX = {}


def pixel_record(t):
    """compact record of a pixel tensor as the model receives it (fp16): shape, per-channel sums and 512 fixed samples"""
    t = torch.as_tensor(t).half().float().reshape(-1, 3, 224, 224)
    n = t.numel()
    if n not in _IDX:
        _IDX[n] = np.random.default_rng(n).choice(n, 512, replace=False)
    return dict(shape=list(t.shape), channel_sums=t.double().sum((0, 2, 3)).tolist(), samples=t.reshape(-1)[_IDX[n]].tolist())


def image_sha(image):
    return hashlib.sha256(np.asarray(image.convert("RGB")).tobytes()).hexdigest() + f":{image.width}x{image.height}"


def array_sha(a):
    return None if a is None else hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest() + ":" + "x".join(map(str, a.shape))
