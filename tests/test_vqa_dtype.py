"""Host-side plumbing of the fp16 SEAL VQA LLM (no GPU): the dtype options are opt-in, validated before anything is loaded,
and every _f16 entry point has the signature of its _bf16 sibling."""
import types

import pytest
import torch


def test_cli_vqa_dtype_flag():
    from vstar_b200.bench_eval import build_parser
    assert build_parser().parse_args([]).vqa_dtype == "bf16"
    assert build_parser().parse_args(["--vqa-dtype", "fp16"]).vqa_dtype == "fp16"
    with pytest.raises(SystemExit):
        build_parser().parse_args(["--vqa-dtype", "fp32"])


def test_dtype_options_are_validated_before_loading():
    from oracle import vsm_oracle as O
    from vstar_b200.engine import CoreWeights, VSMWeights
    from vstar_b200.vqa import VQA_LLM

    def never(name):
        raise AssertionError("no tensor may be read for a rejected dtype")
    cfg = O.tiny_config()
    with pytest.raises(ValueError):
        VSMWeights(cfg, never, device="cpu", dtype=torch.float16)          # the VSM is bf16-only, as in the reference
    with pytest.raises(ValueError):
        CoreWeights(cfg, never, device="cpu", dtype=torch.float32)
    with pytest.raises(ValueError):
        VQA_LLM(types.SimpleNamespace(vqa_model_path="/nonexistent", vqa_dtype="fp32"))


def test_f16_twins_share_the_bf16_signatures():
    from vstar_b200 import _lib
    twins = [n for n in _lib.SIGNATURES if n.endswith("_f16")]
    assert len(twins) == 15
    for n in twins:
        sib = "vsb_llama_layers" if n == "vsb_llama_layers_f16" else n[:-len("_f16")] + "_bf16"
        assert _lib.SIGNATURES[n] == _lib.SIGNATURES[sib], n
