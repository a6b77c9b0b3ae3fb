"""TEST INFRASTRUCTURE ONLY: writes tests/golden/seal_open_golden.json from the REFERENCE's own demo, `inference()` of app.py
(app.py:130-233), run on the six cases of tests/seal_open_helpers.py.

Run where a checkout of the reference is available (oracle/ref_shims.py, VSTAR_REFERENCE_ROOT):

    python -m tools.make_seal_open_golden

Before app.py is imported: the reference modules are made importable by oracle/ref_shims; `gradio` and `bleach` (UI only, not
installed) get test-only stand-in modules; `vstar_bench_eval.VQA_LLM` becomes the reference's own VQA_LLM class with a
character tokenizer, the transformers CLIP image processor and a stub model whose generate() answers from
tests.seal_open_helpers.answer_ids and records what it is handed; `visual_search.VSM` becomes a placeholder, and app.py's
`visual_search` the scripted outcomes of tests.seal_open_helpers.fake_search.  Recorded per case: the four outputs (the
annotated image as a byte hash), every generate() call (input ids, the image the VQA LLM was given, the pixel tensors, the
long/short flags, max_new_tokens, temperature) and every search call.
"""
import contextlib
import io
import json
import os
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_shims, vsm_oracle as O  # noqa: E402
from oracle.make_golden import GOLDEN_DIR, hf_cfgs  # noqa: E402
from tests import seal_open_helpers as H  # noqa: E402

GOLD = os.path.join(GOLDEN_DIR, "seal_open_golden.json")


def _ui_stubs():
    class _Widget:
        def __init__(self, *a, **k):
            pass

        def queue(self, *a, **k):
            return self

        def launch(self, *a, **k):
            return None

    gr = types.ModuleType("gradio")
    gr.Interface = gr.Textbox = gr.Image = _Widget
    sys.modules["gradio"] = gr
    bl = types.ModuleType("bleach")
    bl.clean = lambda s, *a, **k: s
    sys.modules["bleach"] = bl


def main():
    assert ref_shims.reference_available(), "needs a checkout of the reference (VSTAR_REFERENCE_ROOT)"
    ref_shims.install(*hf_cfgs(O.tiny_config()))
    _ui_stubs()
    import torch
    from transformers.models.clip.image_processing_pil_clip import CLIPImageProcessorPil

    import visual_search as RVS          # the reference modules
    import vstar_bench_eval as E

    calls, searches = [], []

    class StubModel:
        def generate(self, input_ids, images=None, object_features=None, images_long=None, objects_long=None, do_sample=False,
                     num_beams=1, temperature=0, top_p=None, max_new_tokens=200, use_cache=True, stopping_criteria=None):
            ids = input_ids.view(-1).tolist()
            calls[-1].update(ids=ids, images=H.pixel_record(images.float()),
                             object_features=None if object_features is None else H.pixel_record(object_features.float()),
                             images_long=images_long, objects_long=objects_long, max_new_tokens=max_new_tokens,
                             temperature=temperature, do_sample=do_sample, num_beams=num_beams)
            return torch.cat([input_ids.cpu(), torch.tensor([H.answer_ids(ids)])], 1)

    class RefVQA(E.VQA_LLM):
        def __init__(self, args):
            self.tokenizer, self.model, self.conv_type = H.CharTokenizer(), StubModel(), args.conv_type
            self.image_processor = CLIPImageProcessorPil()        # transformers' PIL-backed CLIP processor (4.31's behaviour)
            self.image_processor.crop_size = {"height": 224, "width": 224}

        def free_form_inference(self, image, question, **kw):
            calls.append(dict(image=H.image_sha(image), question=question))
            return super().free_form_inference(image, question, **kw)

    E.VQA_LLM = RefVQA
    RVS.VSM = lambda args: object()
    sys.argv = [sys.argv[0]]
    import app as A                      # the reference demo (module level: builds the stub models and the stub UI)

    def search(vsm, image, target_object_name, target_bbox=None, smallest_size=224, confidence_low=None, **kw):
        searches.append(dict(name=target_object_name, image=H.image_sha(image), target_bbox=target_bbox, smallest_size=smallest_size,
                             confidence_low=confidence_low, other=sorted(kw)))
        return H.fake_search(target_object_name, image)

    A.visual_search = search
    out = []
    with tempfile.TemporaryDirectory() as tmp:
        for k, case in enumerate(H.CASES):
            path = os.path.join(tmp, f"case{k}.png")
            H.case_image(case).save(path)
            del calls[:], searches[:]
            with contextlib.redirect_stdout(io.StringIO()):
                res = A.inference(case[0], path)
            assert len(res) == 4, res
            out.append(dict(question=case[0], outputs=[res[0], res[1], H.array_sha(res[2]), res[3]], calls=list(calls),
                            searches=list(searches)))
    with open(GOLD, "w") as f:
        json.dump(dict(cases=out), f, indent=1)
    print(f"{len(out)} cases, {sum(len(c['calls']) for c in out)} generate calls, {sum(len(c['searches']) for c in out)} searches -> {GOLD}")


if __name__ == "__main__":
    main()
