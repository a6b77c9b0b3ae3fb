"""CPU: the VQA oracle (oracle/vqa_oracle.py) against the goldens produced by the REAL reference
LlavaSearchLlamaForCausalLM (oracle/make_golden.py:case_vqa)."""
import os

import numpy as np
import pytest
import torch

from oracle import vqa_oracle as V, vsm_oracle as O
from vstar_b200 import synth

G = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("sub", ["short_long", "long_short"])
def test_vqa_oracle_golden(sub):
    g = np.load(os.path.join(G, f"vqa_a_{sub}.npz"))
    cfg = O.tiny_config()
    sd = {k: synth.synthetic_tensor(k, shp, seed=4321) for k, shp in V.vqa_state_dict_shapes(cfg).items()}
    gen = torch.Generator().manual_seed(int(g["img_seed"]))
    image = torch.randn(1, 3, 224, 224, generator=gen)
    crops = torch.randn(2, 3, 224, 224, generator=gen)
    q = torch.from_numpy(g["q"])
    il, ol = [bool(x) for x in g["images_long"]], [bool(x) for x in g["objects_long"]]
    logits = V.forward_logits(sd, cfg, V.build_embeds(sd, cfg, q, image, crops, il, ol))
    assert logits.shape[1] == int(g["T"])
    assert torch.allclose(logits[0, -1], torch.from_numpy(g["logits_last"]), rtol=1e-4, atol=1e-4)
    assert np.array_equal(logits[0].argmax(-1).numpy(), g["logits_argmax"])
    opts, o = [], 0
    for n in g["opt_lens"]:
        opts.append(torch.from_numpy(g["opts"][o:o + int(n)]))
        o += int(n)
    losses, choice = V.option_losses(sd, cfg, q, opts, image, crops, il, ol)
    assert torch.allclose(losses, torch.from_numpy(g["option_losses"]), rtol=1e-4, atol=1e-4)
    assert choice == int(np.argmin(g["option_losses"]))
    # the as-written variant (question prefilled once, options appended on its past_key_values) gives the same numbers
    losses_c, choice_c = V.option_losses_cached(sd, cfg, q, opts, image, crops, il, ol)
    assert torch.allclose(losses_c, torch.from_numpy(g["option_losses"]), rtol=1e-4, atol=1e-4) and choice_c == choice
    assert V.free_form_generate(sd, cfg, q, image, crops, il, ol, max_new_tokens=4, eos_token_id=-1) == g["gen"].tolist()


def test_tokenizer_image_object_token():
    from vstar_b200.vqa import build_prompt_v1, tokenizer_image_object_token
    from vstar_b200.vsm import SyntheticTokenizer
    tok = SyntheticTokenizer(O.tiny_config())
    p = build_prompt_v1("<image>\nIs the mug <object> at [0.1,0.2,0.3,0.4] next to the cup <object> ?")
    ids = tokenizer_image_object_token(p, tok)
    assert ids[0] == 1 and ids.count(-200) == 1 and ids.count(-300) == 2 and ids.index(-200) < ids.index(-300)
    full = tokenizer_image_object_token(build_prompt_v1("<image>\nq", "yes"), tok)
    assert full[:len(tokenizer_image_object_token(build_prompt_v1("<image>\nq"), tok))] == tokenizer_image_object_token(build_prompt_v1("<image>\nq"), tok)


def test_bf16_vs_fp16_option_choice_bound():
    """The reference runs the SEAL VQA LLM in fp16 (LLaVA/llava/model/builder.py:43, vstar_bench_eval.py:93); the sm_90a kernels
    compute in bf16 with fp32 accumulation.  On the goldens produced by the real reference (fp32), the oracle executed in fp16 and
    in bf16 bounds what the dtype change can do to option scoring: both stay within 2e-2 of the fp32 NLLs, bf16's error is
    within 16x of fp16's (3 fewer mantissa bits), and the chosen option is the fp32 one whenever the two best options are
    further apart than the dtype error - i.e. a choice can only flip inside a near-tie, for either dtype."""
    cfg = O.tiny_config()
    from vstar_b200 import synth
    sd = {k: synth.synthetic_tensor(k, shp, seed=4321) for k, shp in V.vqa_state_dict_shapes(cfg).items()}
    for sub in ("short_long", "long_short"):
        g = np.load(os.path.join(G, f"vqa_a_{sub}.npz"))
        gen = torch.Generator().manual_seed(int(g["img_seed"]))
        image = torch.randn(1, 3, 224, 224, generator=gen)
        crops = torch.randn(2, 3, 224, 224, generator=gen)
        q = torch.from_numpy(g["q"])
        il, ol = [bool(x) for x in g["images_long"]], [bool(x) for x in g["objects_long"]]
        opts, o = [], 0
        for n in g["opt_lens"]:
            opts.append(torch.from_numpy(g["opts"][o:o + int(n)]))
            o += int(n)
        ref = torch.from_numpy(g["option_losses"])
        errs = {}
        for name, dt in (("fp16", torch.float16), ("bf16", torch.bfloat16)):
            sdd = {k: v.to(dt) for k, v in sd.items()}
            losses, choice = V.option_losses_cached(sdd, cfg, q, opts, image.to(dt), crops.to(dt), il, ol)
            errs[name] = float((losses.float() - ref).abs().max())
            srt = ref.sort().values
            if float(srt[1] - srt[0]) > 2 * errs[name]:
                assert choice == int(ref.argmin()), (name, sub)
        # measured on the goldens: fp16 4.5e-4, bf16 5.0e-3 (mean token NLL, values ~6): a bf16 choice can differ from the
        # reference's fp16 choice only when the two best options are within ~1e-2 of each other
        assert errs["fp16"] < 2e-3 and errs["bf16"] < 2e-2, errs
        assert errs["bf16"] <= 16 * errs["fp16"] + 1e-3, errs
