"""CPU oracle of the NF4 weight format of the SEAL VQA LLM's 4-bit mode (the reference's load_4bit: bitsandbytes NF4 with
double-quantised scales, bnb_4bit_compute_dtype fp16; LLaVA/llava/model/builder.py:26-43).

Written from bitsandbytes' published NF4 / double-quant algorithm; this file is the specification the CUDA quantiser
(vstar_b200/csrc/nf4.cu) is tested against bit for bit.  bitsandbytes itself is not a dependency, so equality with the codes
it would produce is not checked here.  Per HF tensor W [out, in]:
  1. blocks of 64 consecutive row-major values, absmax = max |w| (fp32);
  2. code = index of the NF4 entry nearest to w * fp32(1 / absmax) (ties to the lower code; absmax == 0 gives the 0.0 code);
  3. two codes per byte, first element in the high nibble;
  4. double quant: offset = mean(absmax); c = absmax - offset in groups of 256 scales; absmax2 = max |c|;
     q8 = nearest entry of the signed 8-bit dynamic map to c * fp32(1 / absmax2); scale = fp32(fp32(map[q8] * absmax2) + offset);
  5. dequantised weight = fp16(fp32(nf4[code] * scale)).
"""
import numpy as np
import torch

NF4 = np.array([-1.0, -0.6961928009986877, -0.5250730514526367, -0.39491748809814453, -0.28444138169288635, -0.18477343022823334,
                -0.09105003625154495, 0.0, 0.07958029955625534, 0.16093020141124725, 0.24611230194568634, 0.33791524171829224,
                0.44070982131767273, 0.5626170039176941, 0.7229568362236023, 1.0], dtype=np.float32)


def dynamic_map():
    """bitsandbytes create_dynamic_map(signed=True, max_exponent_bits=7, total_bits=8): for i = 0..6 the midpoints of
    linspace(0.1, 1, 2^i + 1) scaled by 10^(i-6), with both signs, plus 0 and 1.0, sorted (fp32, 256 entries)"""
    data = []
    for i in range(7):
        b = torch.linspace(0.1, 1, 2 ** i + 1)
        means = (b[:-1] + b[1:]) / 2.0
        scale = 10 ** (i - 6)
        data += (scale * means).tolist() + (-scale * means).tolist()
    data += [0.0, 1.0]
    return np.array(sorted(data), dtype=np.float32)


def _recip(a):
    a = np.asarray(a, dtype=np.float32)
    with np.errstate(divide="ignore"):
        return np.where(a > 0, np.float32(1.0) / np.where(a > 0, a, np.float32(1.0)), np.float32(0.0)).astype(np.float32)


def _nearest(v, table, chunk=1 << 20):
    """index of the nearest table entry (fp32 distances, first index on ties) for every value of v (1-D fp32)"""
    out = np.empty(v.shape, dtype=np.int64)
    for s in range(0, v.size, chunk):
        d = np.abs(v[s:s + chunk, None] - table[None, :])
        out[s:s + chunk] = d.argmin(1)
    return out


def quantize(w, offset=None):
    """w fp16 [N, K] (numpy or torch), K % 64 == 0 -> (codes uint8 [N, K/2], absmax fp32 [N, K/64], scales fp32 [N, K/64]).
    offset: the double-quant offset (default: mean of absmax; the device quantiser takes torch's mean on the GPU, pass that one to
    compare bit for bit)."""
    w = np.asarray(w.cpu().numpy() if isinstance(w, torch.Tensor) else w, dtype=np.float16)
    N, K = w.shape
    assert K % 64 == 0, K
    blocks = w.astype(np.float32).reshape(-1, 64)
    absmax = np.abs(blocks).max(1).astype(np.float32)
    v = (blocks * _recip(absmax)[:, None]).astype(np.float32)
    idx = _nearest(v.reshape(-1), NF4).reshape(-1, 2)
    codes = ((idx[:, 0] << 4) | idx[:, 1]).astype(np.uint8).reshape(N, K // 2)
    if offset is None:
        offset = np.float32(torch.from_numpy(absmax).mean().item())
    offset = np.float32(offset)
    n = absmax.size
    c = (absmax - offset).astype(np.float32)
    pad = (-n) % 256
    cg = np.concatenate([c, np.zeros(pad, np.float32)]).reshape(-1, 256)
    am2 = np.abs(cg).max(1).astype(np.float32)
    dmap = dynamic_map()
    q8 = _nearest((cg * _recip(am2)[:, None]).astype(np.float32).reshape(-1), dmap).reshape(cg.shape)
    scales = ((dmap[q8] * am2[:, None]).astype(np.float32) + offset).astype(np.float32).reshape(-1)[:n]
    return codes, absmax.reshape(N, K // 64), scales.reshape(N, K // 64)


def dequantize(codes, scales):
    """(codes uint8 [N, K/2], scales fp32 [N, K/64]) -> fp16 [N, K]"""
    codes = np.asarray(codes, dtype=np.uint8)
    N = codes.shape[0]
    K = codes.shape[1] * 2
    idx = np.stack([codes >> 4, codes & 15], -1).reshape(N, K)
    s = np.repeat(np.asarray(scales, dtype=np.float32), 64, axis=1)
    return (NF4[idx] * s).astype(np.float32).astype(np.float16)


def quantized_keys(sd):
    """names of the state-dict tensors the 4-bit mode quantises: every nn.Linear weight of the Llama layers, mm_projector and
    mm_projector_object (perceiver to_q / to_kv / to_out, its feed-forward Linears, the final Linear); not lm_head, embeddings,
    norms, biases, latents or the CLIP tower"""
    keys = []
    for k in sd:
        if not k.endswith(".weight") or "vision_tower" in k:
            continue
        if k.startswith("model.layers.") and (".self_attn." in k or ".mlp." in k):
            keys.append(k)
        elif k == "model.mm_projector.weight" or k == "model.mm_projector_object.2.weight":
            keys.append(k)
        elif k.startswith("model.mm_projector_object.1.layers.") and (k.endswith((".to_q.weight", ".to_kv.weight", ".to_out.weight"))
                                                                     or k.endswith((".1.1.weight", ".1.3.weight"))):
            keys.append(k)
    return keys


def dequantized_state_dict(sd):
    """copy of a VQA state dict whose quantised Linear weights are replaced by their fp16 NF4 round trip: oracle/vqa_oracle.py on
    it computes the reference's 4-bit model"""
    out = dict(sd)
    for k in quantized_keys(sd):
        w = sd[k]
        codes, _, scales = quantize(w.to(torch.float16))
        out[k] = torch.from_numpy(dequantize(codes, scales)).to(w.dtype)
    return out
