"""The pipelined open-ended SEAL answering (seal.answer_open_stream) on the GPU: in batch-invariant mode it equals the phased
answer_open_many item by item, on all four outputs (the annotated image byte for byte), greedy on the contiguous stream, with
kv_pages, kv_pages + kv_swap_pages and kv_pages + prefill_chunk, and beam-searched (num_beams = 2) on the bf16 engine, and
greedy on the fp16 and NF4 engines; sampled runs repeat under the same torch.manual_seed; a request the pool cannot hold
raises ValueError and leaves no device memory behind.  The setup is test_vqa_stream_gpu's answer_open_many test: the tiny
synthetic VSM, a scripted LLM whose direct answers name missing objects, and confidence_high = 2.0."""
import gc
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MISSING = {0: ["mug", "cup"], 2: ["dog"], 3: ["a", "b", "c"], 4: ["pen"]}
KW = dict(minimum_size=128, search_batch=4, search_kwargs=dict(confidence_high=2.0))


@pytest.fixture(scope="module")
def ops():
    from vstar_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def setup():
    from oracle import vqa_oracle as V, vsm_oracle as O
    from PIL import Image
    from tests.helpers import FakeNLP
    from vstar_b200 import noun_chunks, synth
    from vstar_b200.engine import VSMEngine, VSMWeights
    from vstar_b200.vsm import VSM
    cfg = O.tiny_config()
    sd = {k: synth.synthetic_tensor(k, shp, seed=4321) for k, shp in V.vqa_state_dict_shapes(cfg).items()}
    j = json.load(open(os.path.join(ROOT, "tests", "golden", "tiny_config.json")))
    vcfg = O.VSMConfig(**j["cfg"])
    vsm_eng = VSMEngine(VSMWeights.from_state_dict(vcfg, O.synthetic_state_dict(vcfg, seed=j["weight_seed"])))
    prompt, ans = O.synthetic_prompt(vcfg, n_text=24, seed=11)
    noun_chunks.set_nlp(FakeNLP())                # the weak-cue branch's noun chunker (spaCy is not a test dependency)

    class TinyVSM(VSM):
        def _ids(self, question):
            return prompt[0].tolist()

    vsm = TinyVSM(engine=vsm_eng, forced_answer_ids=ans.tolist(), frontier_batch=4)
    rng = np.random.default_rng(8)
    items = [(Image.fromarray(rng.integers(0, 256, (200 + 30 * i, 260, 3), dtype=np.uint8), "RGB"), f"what is in image {i}")
             for i in range(6)]
    yield cfg, sd, vsm, items
    noun_chunks.set_nlp(None)


_LLMS = {}


def scripted_llm(setup, kind):
    """VQA_LLM whose direct answers name MISSING's objects (random weights never do) on both decode paths; final answers
    are the model's own"""
    from vstar_b200 import seal
    from vstar_b200.vqa import VQA_LLM, AnswerSession, VQAEngine, VQAWeights
    if kind in _LLMS:
        return _LLMS[kind]
    cfg, sd, _, _ = setup

    def script(i, text):
        return seal.MISSING_OBJECTS_MSG + " " + ", ".join(MISSING[i]) + "." if i in MISSING else text

    class ScriptedSession(AnswerSession):
        def step(self):
            return [((i, stage), script(i, text) if stage == 0 else text) for (i, stage), text in super().step()]

    class ScriptedLLM(VQA_LLM):
        def free_form_inference_stream(self, items, *a, **kw):
            for i, text in super().free_form_inference_stream(items, *a, **kw):
                q = items[i][1]
                yield i, text if seal.FOCUS_MSG in q else script(int(q.split()[-1]), text)

        def answer_session(self, max_new_tokens, slots, max_positions=None, num_beams=1, **kw):
            return ScriptedSession(self, max_new_tokens, slots, max_positions or self.engine.MAX_POSITIONS, num_beams, **kw)

    w = dict(bf16={}, fp16=dict(dtype=torch.float16), nf4=dict(dtype=torch.float16, quant="nf4"))[kind]
    _LLMS[kind] = ScriptedLLM(engine=VQAEngine(VQAWeights.from_state_dict(cfg, sd, **w), max_tokens=1024))
    return _LLMS[kind]


def keyed(outs):
    return [(o[0], o[1], None if o[2] is None else (o[2].shape, o[2].tobytes()), o[3]) for o in outs]


def pipelined(llm, vsm, items, **kw):
    from vstar_b200 import seal
    out = [None] * len(items)
    order = []
    for i, o in seal.answer_open_stream(llm, vsm, items, **kw):
        assert out[i] is None
        out[i], _ = o, order.append(i)
    return out, order


CASES = [("bf16", {}), ("bf16", dict(kv_pages=48)), ("bf16", dict(kv_pages=24, kv_swap_pages=64)),
         ("bf16", dict(kv_pages=48, prefill_chunk=64)), ("bf16", dict(num_beams=2, slots=4)), ("fp16", {}), ("nf4", {})]


@pytest.mark.parametrize("kind,kw", CASES, ids=[f"{k}-{'-'.join(map(str, kw.items())) or 'contiguous'}" for k, kw in CASES])
def test_answer_open_stream_equals_answer_open_many(setup, ops, kind, kw):
    from vstar_b200 import seal
    _, _, vsm, items = setup
    llm = scripted_llm(setup, kind)
    kw = dict(dict(slots=3, searches_in_flight=3), **kw, **KW)
    with ops.batch_invariant():
        many = seal.answer_open_many(llm, vsm, items, **kw)
        got, order = pipelined(llm, vsm, items, **kw)
    assert keyed(got) == keyed(many)
    assert [o[1:] == (None, None, None) for o in got] == [i not in MISSING for i in range(len(items))]
    assert sorted(order) == list(range(len(items)))


def test_sampled_pipeline_repeats_under_the_seed(setup, ops):
    _, _, vsm, items = setup
    llm = scripted_llm(setup, "bf16")
    runs = []
    with ops.batch_invariant():
        for _ in range(2):
            torch.manual_seed(1234)
            runs.append(keyed(pipelined(llm, vsm, items, slots=3, temperature=0.7, top_p=0.9, **KW)[0]))
    assert runs[0] == runs[1]


def test_request_too_large_for_the_pool_raises_and_frees(setup, ops):
    _, _, vsm, items = setup
    llm = scripted_llm(setup, "bf16")
    list(pipelined(llm, vsm, items[:1], kv_pages=48, **KW))          # warm: layer tables and lazily built engine state
    gc.collect()
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match=r"kv_pages = 2 cannot hold the answer to question 0 \('what is in image 0'\)"):
        pipelined(llm, vsm, items, kv_pages=2, **KW)
    gc.collect()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == m0
