"""ORACLE SUPPORT — TEST INFRASTRUCTURE ONLY (build container only: needs /root/reference).

Lets the UNMODIFIED ``proteingym/baselines/protgpt2/compute_fitness.py`` run ``main()`` on the CPU under the installed transformers:
  * ``Module.cuda()`` and ``Tensor.to("cuda...")`` are no-ops (the script moves the model and every input to cuda:0);
  * ``AutoTokenizer`` in the script's namespace loads the fixture tokenizer (tests/golden/protgpt2_tokenizer, or the folder given to
    ``install``) whatever path it is asked for: the script hard-codes a cluster directory (:77).
The model is transformers' own GPT2LMHeadModel, built by the script's ``AutoModelForCausalLM.from_pretrained``. Nothing is copied from the
reference."""
from __future__ import annotations

import importlib.util
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(os.environ.get("PG_REFERENCE_ROOT", "/root/reference"), "proteingym", "baselines", "protgpt2")
FIXTURE_TOKENIZER = os.path.join(ROOT, "tests", "golden", "protgpt2_tokenizer")


def available() -> bool:
    return os.path.isfile(os.path.join(REF, "compute_fitness.py"))


def install(tokenizer_dir: str = FIXTURE_TOKENIZER):
    """-> the reference ``compute_fitness`` module, importable and CPU-bound."""
    if "compute_fitness_protgpt2" in sys.modules:
        return sys.modules["compute_fitness_protgpt2"]
    import torch
    from transformers import AutoTokenizer
    torch.nn.Module.cuda = lambda self, *a, **k: self
    orig_to = torch.Tensor.to

    def to(self, *args, **kwargs):
        if args and str(args[0]).startswith("cuda"):
            return self
        return orig_to(self, *args, **kwargs)
    torch.Tensor.to = to
    spec = importlib.util.spec_from_file_location("compute_fitness_protgpt2", os.path.join(REF, "compute_fitness.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules["compute_fitness_protgpt2"] = mod
    spec.loader.exec_module(mod)

    class FixtureTokenizer:
        @staticmethod
        def from_pretrained(path, *a, **k):
            return AutoTokenizer.from_pretrained(tokenizer_dir)
    mod.AutoTokenizer = FixtureTokenizer
    return mod
