"""TEST INFRASTRUCTURE ONLY — import shims for the read-only reference tree.

This module exists so that, where a checkout of the reference is available
(VSTAR_REFERENCE_ROOT), the reference's own Python code can be imported under the installed
transformers 5.5 / torch 2.11 and used to (a) validate the CPU restatement in
`oracle/vsm_oracle.py` and (b) generate the golden vectors committed under
`tests/golden/` (see `oracle/make_golden.py`).

Nothing under `vstar_b200/` may import this file.  The tests, smoke() and bench.py
never import it either: they read the committed goldens.

Shims (SURVEY.md §8c):
  1. AutoConfig.register / AutoModelForCausalLM.register -> exist_ok=True
     (reference: VisualSearch/model/llava/model/language_model/llava_llama.py:166-167
      collides with transformers-5 built-in "llava").
  2. sys.modules stubs for the unused MPT branch, spaCy, matplotlib.
  3. torch.Tensor.cuda -> identity, torch.cuda.empty_cache -> no-op (hard-coded
     .cuda() at VisualSearch/model/VSM.py:226,232,302,469,495).
  4. OwlViTConfig.from_pretrained / CLIPVisionConfig.from_pretrained /
     CLIPVisionModel.from_pretrained / CLIPImageProcessor.from_pretrained are
     redirected to in-memory configs (no HF hub, no checkpoints offline).
"""
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("VSTAR_REFERENCE_ROOT", "/root/reference")

_installed = False
_owl_cfg_kwargs = None
_clip_cfg_kwargs = None


def reference_available() -> bool:
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "VisualSearch"))


def install(owl_cfg: dict, clip_cfg: dict):
    """Install the shims.  `owl_cfg` / `clip_cfg` are the HF config kwargs the
    redirected from_pretrained calls will return (lets goldens use tiny models)."""
    global _installed, _owl_cfg_kwargs, _clip_cfg_kwargs
    _owl_cfg_kwargs, _clip_cfg_kwargs = owl_cfg, clip_cfg
    if _installed:
        return
    import torch
    import transformers
    from transformers import AutoConfig, AutoModelForCausalLM

    # (1) register(exist_ok=True)
    _cfg_reg = AutoConfig.register
    _mdl_reg = AutoModelForCausalLM.register

    def cfg_register(model_type, config, exist_ok=False):
        return _cfg_reg(model_type, config, exist_ok=True)

    def mdl_register(config_class, model_class, exist_ok=False):
        return _mdl_reg(config_class, model_class, exist_ok=True)

    AutoConfig.register = staticmethod(cfg_register)
    AutoModelForCausalLM.register = classmethod(lambda cls, c, m, exist_ok=False: _mdl_reg(c, m, exist_ok=True))

    # (2) stubs
    def stub(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    class _Dummy:
        def __init__(self, *a, **k):
            pass

    stub("VisualSearch.model.llava.model.language_model.llava_mpt",
         LlavaMPTConfig=_Dummy, LlavaMPTForCausalLM=_Dummy)
    stub("LLaVA.llava.model.language_model.llava_mpt", LlavaMPTConfig=_Dummy, LlavaMPTForCausalLM=_Dummy)
    try:
        import einops_exts  # noqa: F401
    except Exception:
        import einops
        stub("einops_exts",
             rearrange_many=lambda ts, pattern, **kw: tuple(einops.rearrange(t, pattern, **kw) for t in ts),
             repeat_many=lambda ts, pattern, **kw: tuple(einops.repeat(t, pattern, **kw) for t in ts))
    if "spacy" not in sys.modules:
        try:
            import spacy  # noqa: F401
        except Exception:
            stub("spacy", load=lambda *_a, **_k: (lambda text: []))
    if "matplotlib" not in sys.modules:
        try:
            import matplotlib  # noqa: F401
        except Exception:
            mp = stub("matplotlib")
            mp.pyplot = stub("matplotlib.pyplot")
    try:
        import tqdm  # noqa: F401
    except Exception:
        stub("tqdm", tqdm=lambda x, **k: x)

    # (3) CPU runs
    if not torch.cuda.is_available():
        torch.Tensor.cuda = lambda self, *a, **k: self
        torch.nn.Module.cuda = lambda self, *a, **k: self
        torch.cuda.empty_cache = lambda: None

    # (4) config / model redirection
    from transformers import (CLIPImageProcessor, CLIPVisionConfig,
                              CLIPVisionModel, OwlViTConfig)

    def owl_from_pretrained(cls, name, *a, **k):
        return OwlViTConfig(**_owl_cfg_kwargs)

    def clipcfg_from_pretrained(cls, name, *a, **k):
        return CLIPVisionConfig(**_clip_cfg_kwargs)

    def clipmodel_from_pretrained(cls, name, *a, **k):
        return CLIPVisionModel(CLIPVisionConfig(**_clip_cfg_kwargs))

    def clipproc_from_pretrained(cls, name, *a, **k):
        return CLIPImageProcessor()

    OwlViTConfig.from_pretrained = classmethod(owl_from_pretrained)
    CLIPVisionConfig.from_pretrained = classmethod(clipcfg_from_pretrained)
    CLIPVisionModel.from_pretrained = classmethod(clipmodel_from_pretrained)
    CLIPImageProcessor.from_pretrained = classmethod(clipproc_from_pretrained)

    # (5) transformers-5.5 output-capture drift: once another vision model (OWL-ViT)
    # has run, the capture hooks end up installed twice on the CLIP encoder layers
    # and `hidden_states` contains every layer output twice (7 entries for 3
    # layers).  Under the reference's pinned transformers 4.31 `hidden_states` is
    # (embeddings, layer_1, ..., layer_L); restore that by dropping consecutive
    # entries that are the *same tensor object*.
    _clip_fwd = CLIPVisionModel.forward

    def clip_forward(self, *a, **k):
        out = _clip_fwd(self, *a, **k)
        hs = getattr(out, "hidden_states", None)
        if hs is not None:
            ded = [hs[0]]
            for t in hs[1:]:
                if t is not ded[-1]:
                    ded.append(t)
            out["hidden_states"] = tuple(ded)
        return out

    CLIPVisionModel.forward = clip_forward

    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    _installed = True
