"""The NF4 format of the SEAL VQA LLM's 4-bit mode on the CPU (no GPU): the oracle's tables, nibble order, error bound and
per-tensor quantisation under the fused row layouts, and the load_4bit / --vqa-load-4bit option plumbing."""
import types

import numpy as np
import pytest
import torch

from oracle import nf4_oracle as N


def test_nf4_table_and_nibble_order():
    assert N.NF4.shape == (16,) and N.NF4[0] == -1.0 and N.NF4[7] == 0.0 and N.NF4[15] == 1.0
    assert np.all(np.diff(N.NF4) > 0)
    w = np.zeros((1, 64), np.float16)
    w[0, 0], w[0, 1] = -1.0, 1.0                 # codes 0 and 15 in the first byte: high nibble = first element
    codes, absmax, scales = N.quantize(w)
    assert codes.shape == (1, 32) and codes[0, 0] == 0x0F and np.all(codes[0, 1:] == 0x77)
    assert absmax[0, 0] == 1.0
    deq = N.dequantize(codes, scales)
    assert deq[0, 0] == -scales[0, 0].astype(np.float16) and np.all(deq[0, 2:] == 0)


def test_dynamic_map():
    m = N.dynamic_map()
    assert m.shape == (256,) and m.dtype == np.float32
    assert np.all(np.diff(m) >= 0) and 0.0 in m and 1.0 in m
    assert np.array_equal(np.sort(-m[(m != 0) & (m != 1)]), m[(m != 0) & (m != 1)])     # symmetric apart from 0 and 1
    assert m[0] < 0 and np.count_nonzero(m == 0) == 1


def test_quantize_dequantize_error_bound():
    rng = np.random.default_rng(0)
    w = (rng.standard_normal((96, 256)) * 0.05).astype(np.float16)
    codes, absmax, scales = N.quantize(w)
    deq = N.dequantize(codes, scales).astype(np.float32)
    # per block: half the largest gap of the NF4 table times absmax, plus the double-quant error of the scale
    half_gap = float(np.diff(N.NF4).max()) / 2
    a = np.repeat(absmax, 64, axis=1)
    s = np.repeat(scales, 64, axis=1)
    bound = half_gap * a + np.abs(s - a) + 2 ** -10 * np.abs(deq)
    assert np.all(np.abs(deq - w.astype(np.float32)) <= bound)
    assert np.abs(scales - absmax).max() <= 0.01 * absmax.max()
    assert np.all(N.dequantize(*N.quantize(np.zeros((2, 64), np.float16))[::2]) == 0)


def test_per_tensor_quantisation_commutes_with_the_fused_layouts():
    """quantising q, k, v (gate, up) one by one and concatenating (interleaving) the codes and scales row-wise dequantises to the
    same rows as each tensor's own dequantisation in the fused order"""
    rng = np.random.default_rng(1)
    d, inter = 128, 192
    parts = [(rng.standard_normal((d, d)) * s).astype(np.float16) for s in (0.02, 0.05, 0.1)]
    qs = [N.quantize(p) for p in parts]
    codes = np.concatenate([q[0] for q in qs], 0)
    scales = np.concatenate([q[2] for q in qs], 0)
    assert np.array_equal(N.dequantize(codes, scales), np.concatenate([N.dequantize(q[0], q[2]) for q in qs], 0))
    gate, up = [(rng.standard_normal((inter, d)) * s).astype(np.float16) for s in (0.03, 0.07)]
    qg, qu = N.quantize(gate), N.quantize(up)
    codes = np.stack([qg[0], qu[0]], 1).reshape(2 * inter, -1)
    scales = np.stack([qg[2], qu[2]], 1).reshape(2 * inter, -1)
    dg, du = N.dequantize(qg[0], qg[2]), N.dequantize(qu[0], qu[2])
    deq = N.dequantize(codes, scales)
    assert np.array_equal(deq[0::2], dg) and np.array_equal(deq[1::2], du)
    # the offset and 256-groups are per tensor: quantising the fused matrix instead gives other scales
    assert not np.array_equal(N.quantize(np.concatenate(parts, 0))[2], np.concatenate([q[2] for q in qs], 0))


def test_quantized_keys_of_the_vqa_state_dict():
    from oracle import vqa_oracle as V, vsm_oracle as O
    cfg = O.tiny_config()
    keys = V.vqa_state_dict_shapes(cfg)
    q = set(N.quantized_keys(keys))
    assert "model.layers.0.self_attn.q_proj.weight" in q and "model.layers.0.mlp.down_proj.weight" in q
    assert {"model.mm_projector.weight", "model.mm_projector_object.2.weight", "model.mm_projector_object.1.layers.0.0.to_kv.weight",
            "model.mm_projector_object.1.layers.5.1.1.weight", "model.mm_projector_object.1.layers.5.1.3.weight"} <= q
    for k in q:
        assert "norm" not in k and "lm_head" not in k and "embed" not in k and "vision_tower" not in k and "latents" not in k
        assert keys[k][-1] % 64 == 0, (k, keys[k])
    assert len(q) == 7 * cfg.n_layers + 2 + 6 * 5


def test_load_4bit_options_are_validated_before_loading():
    from vstar_b200.engine import VSMWeights
    from vstar_b200.vqa import VQAWeights, load_pretrained_model
    from oracle import vsm_oracle as O

    def never(name):
        raise AssertionError("no tensor may be read for a rejected option")
    with pytest.raises(ValueError):
        load_pretrained_model("/nonexistent", load_4bit=True, torch_dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError):
        load_pretrained_model("/nonexistent", load_8bit=True)
    cfg = O.tiny_config()
    with pytest.raises(ValueError):
        VQAWeights(cfg, never, device="cpu", quant="nf4")                            # bf16 + NF4
    with pytest.raises(ValueError):
        VQAWeights(cfg, never, device="cpu", dtype=torch.float16, quant="int8")
    with pytest.raises(ValueError):
        VSMWeights(cfg, never, device="cpu", quant="nf4")


def test_cli_vqa_load_4bit_flag(monkeypatch):
    from vstar_b200 import vqa
    from vstar_b200.bench_eval import build_parser
    assert build_parser().parse_args([]).vqa_load_4bit is False
    args = build_parser().parse_args(["--vqa-load-4bit", "--vqa-model-path", "/ckpt"])
    assert args.vqa_load_4bit is True
    seen = {}

    def fake_load(path, base, name, load_8bit=False, load_4bit=False, torch_dtype=None, **kw):
        seen.update(path=path, load_4bit=load_4bit, torch_dtype=torch_dtype)
        raise RuntimeError("stop")
    monkeypatch.setattr(vqa, "load_pretrained_model", fake_load)
    with pytest.raises(RuntimeError):
        vqa.VQA_LLM(args)
    assert seen == dict(path="/ckpt", load_4bit=True, torch_dtype=None)
    with pytest.raises(RuntimeError):
        vqa.VQA_LLM(types.SimpleNamespace(vqa_model_path="/ckpt", vqa_dtype="fp16"))
    assert seen == dict(path="/ckpt", load_4bit=False, torch_dtype=torch.float16)
