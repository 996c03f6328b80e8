"""ORACLE SUPPORT — TEST INFRASTRUCTURE ONLY (build container only: needs /root/reference).

Lets the UNMODIFIED ``ProGen3ForCausalLM`` and ``ProGen3Scorer`` (proteingym/baselines/progen3/progen3/) run on the CPU in fp32 under the
installed packages, through five import shims:
  1. stub packages ``megablocks`` and ``megablocks.layers.{moe,dmoe,arguments,common}``, each submodule set as an attribute of its parent;
     they are only imported: the "eager" MoE never calls them;
  2. ``flash_attn.ops.triton.layer_norm.rms_norm_fn`` as plain torch, ``x.float() * rsqrt(mean(x^2) + eps) * w`` cast back to the input
     dtype, installed AFTER transformers is imported (its flash-attn probe fails on a module without a spec);
  3. a stub ``Bio.SeqIO`` (imported by scorer.py; the goldens call ``evaluate``, not ``run``);
  4. ``transformers.modeling_utils.GenerationMixin`` pointed at ``transformers.generation.GenerationMixin`` (moved in transformers 5);
  5. ``DynamicCache.from_legacy_cache = classmethod(lambda cls, pkv=None: cls())`` (dropped in transformers 5; use_cache defaults on).
SDPA with the FLASH_ATTENTION backend runs fp32 on the CPU. Nothing is copied from the reference."""
from __future__ import annotations

import os
import sys
import types

REF = os.path.join(os.environ.get("PG_REFERENCE_ROOT", "/root/reference"), "proteingym", "baselines", "progen3")


def available() -> bool:
    return os.path.isfile(os.path.join(REF, "progen3", "modeling.py"))


def _module(name: str, package: bool = False):
    m = types.ModuleType(name)
    if package:
        m.__path__ = []
    sys.modules[name] = m
    return m


def install():
    import torch
    import transformers  # noqa: F401  (before the flash_attn stub)
    import transformers.modeling_utils as mu
    from transformers import generation
    from transformers.cache_utils import DynamicCache
    if "megablocks" not in sys.modules:
        mb = _module("megablocks", True)
        layers = _module("megablocks.layers", True)
        mb.layers = layers
        for sub in ("moe", "dmoe", "arguments", "common"):
            setattr(layers, sub, _module(f"megablocks.layers.{sub}"))
        layers.arguments.Arguments = lambda *a, **k: None
        layers.dmoe.dMoE = type("dMoE", (), {})
    if "flash_attn.ops.triton.layer_norm" not in sys.modules:
        fa = _module("flash_attn", True)
        ops = _module("flash_attn.ops", True)
        tri = _module("flash_attn.ops.triton", True)
        ln = _module("flash_attn.ops.triton.layer_norm")
        fa.ops, ops.triton, tri.layer_norm = ops, tri, ln

        def rms_norm_fn(x, weight, bias=None, residual=None, eps=1e-6, **kw):
            y = x.float() * torch.rsqrt(x.float().pow(2).mean(-1, keepdim=True) + eps) * weight.float()
            return y.to(x.dtype)
        ln.rms_norm_fn = rms_norm_fn
    if "Bio.SeqIO" not in sys.modules:
        bio = _module("Bio", True)
        bio.SeqIO = _module("Bio.SeqIO")
    if not hasattr(mu, "GenerationMixin"):
        mu.GenerationMixin = generation.GenerationMixin
    if not hasattr(DynamicCache, "from_legacy_cache"):
        DynamicCache.from_legacy_cache = classmethod(lambda cls, pkv=None: cls())
    if REF not in sys.path:
        sys.path.insert(0, REF)


def load_model(cfg: dict, state: dict):
    """The reference ProGen3ForCausalLM (fp32, eager MoE) with the eager-layout ``state``."""
    install()
    from progen3.config import ProGen3Config
    from progen3.modeling import ProGen3ForCausalLM
    conf = ProGen3Config(**{k: v for k, v in cfg.items() if k != "model_type"})
    m = ProGen3ForCausalLM(conf)
    missing, unexpected = m.load_state_dict(state, strict=False)
    if missing or unexpected:
        raise RuntimeError(f"state dict mismatch: missing {missing}, unexpected {unexpected}")
    return m.float().eval()


def scorer(model, max_batch_tokens: int = 65536):
    install()
    from progen3.scorer import ProGen3Scorer
    return ProGen3Scorer(model, max_batch_tokens=max_batch_tokens)
