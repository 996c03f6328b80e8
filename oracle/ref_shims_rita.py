"""ORACLE SUPPORT — TEST INFRASTRUCTURE ONLY (build container only: needs /root/reference).

Lets the UNMODIFIED ``proteingym/baselines/rita/compute_fitness.py`` run ``main()`` on the CPU:
  * ``AutoModelForCausalLM`` in the script's namespace builds ``RITAModelForCausalLM`` from the reference's own ``rita_modeling.py`` /
    ``rita_configuration.py`` (imported as a package) and loads the directory's state dict strictly; the output head is tied to the
    embedding explicitly when config.json does not set ``tie_word_embeddings`` to false, so the goldens do not depend on what the
    installed transformers release does about tying;
  * ``AutoTokenizer`` in the script's namespace ignores the hard-coded cluster path (:75) and loads ``TOKENIZER_DIR`` with the installed
    transformers' ``AutoTokenizer``;
  * ``Module.cuda()`` and ``Tensor.to("cuda...")`` are no-ops (the script moves the model and every input to cuda:0).
Nothing is copied from the reference."""
from __future__ import annotations

import importlib.util
import json
import os
import sys

REF = os.path.join(os.environ.get("PG_REFERENCE_ROOT", "/root/reference"), "proteingym", "baselines", "rita")
TOKENIZER_DIR = None  # set by the caller before main() runs


def available() -> bool:
    return os.path.isfile(os.path.join(REF, "compute_fitness.py"))


def _package():
    if "rita_ref" in sys.modules:
        return sys.modules["rita_ref"]
    import importlib.machinery
    import types
    pkg = types.ModuleType("rita_ref")  # a namespace for the reference's two modules (rita_modeling imports .rita_configuration)
    pkg.__path__ = [REF]
    pkg.__spec__ = importlib.machinery.ModuleSpec("rita_ref", None, is_package=True)
    pkg.__spec__.submodule_search_locations = [REF]
    sys.modules["rita_ref"] = pkg
    return pkg


def load_model(folder: str):
    """RITAModelForCausalLM of the reference, weights from ``folder`` (strict), head tied per config.json."""
    import torch
    _package()
    from rita_ref.rita_configuration import RITAConfig
    from rita_ref.rita_modeling import RITAModelForCausalLM
    cfg = json.load(open(os.path.join(folder, "config.json")))
    tied = bool(cfg.get("tie_word_embeddings", True))
    conf = RITAConfig(**{k: v for k, v in cfg.items() if k not in ("model_type", "tie_word_embeddings")})
    m = RITAModelForCausalLM(conf)
    st = torch.load(os.path.join(folder, "pytorch_model.bin"), map_location="cpu", weights_only=True)
    m.load_state_dict(st, strict=True)
    if tied:
        m.lm_head.weight = m.transformer.embedding.weight
    return m.eval()


class _AutoModel:
    @staticmethod
    def from_pretrained(path, **kw):
        return load_model(path)


class _AutoTokenizer:
    @staticmethod
    def from_pretrained(path, **kw):
        from transformers import AutoTokenizer
        return AutoTokenizer.from_pretrained(TOKENIZER_DIR)


def install():
    """-> the reference ``compute_fitness`` module, importable and CPU-bound."""
    if "compute_fitness_rita" in sys.modules:
        return sys.modules["compute_fitness_rita"]
    import torch
    torch.nn.Module.cuda = lambda self, *a, **k: self
    orig_to = torch.Tensor.to

    def to(self, *args, **kwargs):
        if args and str(args[0]).startswith("cuda"):
            return self
        return orig_to(self, *args, **kwargs)
    torch.Tensor.to = to
    spec = importlib.util.spec_from_file_location("compute_fitness_rita", os.path.join(REF, "compute_fitness.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules["compute_fitness_rita"] = mod
    spec.loader.exec_module(mod)
    mod.AutoModelForCausalLM = _AutoModel
    mod.AutoTokenizer = _AutoTokenizer
    return mod
