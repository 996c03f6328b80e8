"""ORACLE SUPPORT — TEST INFRASTRUCTURE ONLY (build container only: needs /root/reference).

Lets the UNMODIFIED ``proteingym/baselines/progen2/compute_fitness.py`` run ``main()`` on the CPU under the installed transformers:
  * a stub module ``transformers.utils.model_parallel_utils`` (``assert_device_map`` / ``get_device_map``, imported by
    modeling_progen.py but used only by ``parallelize``);
  * ``init_weights`` is a no-op on ``ProGenModel`` / ``ProGenForCausalLM`` (the weights are loaded right after), and
    ``ProGenModel.get_head_mask`` returns one ``None`` per layer (the reference never passes a head mask);
  * ``create_model`` in the script's namespace builds ``ProGenForCausalLM`` from the directory's config.json and loads its
    pytorch_model.bin strictly (the attention mask buffers excepted, which the model builds itself), instead of
    ``from_pretrained``; ``--fp16`` is not used by the goldens;
  * ``Module.cuda()`` and ``Tensor.to("cuda...")`` are no-ops (the script moves the model and every input to cuda:0).
The tokenizer is the reference's own ``tokenizer.json``, read by the script through the installed ``tokenizers``.
Nothing is copied from the reference."""
from __future__ import annotations

import importlib.util
import json
import os
import sys
import types

REF = os.path.join(os.environ.get("PG_REFERENCE_ROOT", "/root/reference"), "proteingym", "baselines", "progen2")


def available() -> bool:
    return os.path.isfile(os.path.join(REF, "compute_fitness.py"))


def _model_module():
    if "transformers.utils.model_parallel_utils" not in sys.modules:
        stub = types.ModuleType("transformers.utils.model_parallel_utils")
        stub.assert_device_map = lambda *a, **k: None
        stub.get_device_map = lambda *a, **k: None
        sys.modules["transformers.utils.model_parallel_utils"] = stub
    if REF not in sys.path:
        sys.path.insert(0, REF)
    from models.progen import modeling_progen as M
    M.ProGenModel.init_weights = lambda self, *a, **k: None
    M.ProGenForCausalLM.init_weights = lambda self, *a, **k: None
    M.ProGenModel.get_head_mask = lambda self, hm, n, *a, **k: [None] * n
    return M


def load_model(folder: str):
    """ProGenForCausalLM of the reference with the weights of ``folder`` (config.json + pytorch_model.bin)."""
    import torch
    M = _model_module()
    from models.progen.configuration_progen import ProGenConfig
    cfg = json.load(open(os.path.join(folder, "config.json")))
    conf = ProGenConfig(**{k: v for k, v in cfg.items() if k != "model_type"})
    m = M.ProGenForCausalLM(conf)
    st = torch.load(os.path.join(folder, "pytorch_model.bin"), map_location="cpu", weights_only=True)
    missing, unexpected = m.load_state_dict(st, strict=False)
    missing = [k for k in missing if not (k.endswith("attn.bias") or k.endswith("attn.masked_bias"))]
    if missing or unexpected:
        raise RuntimeError(f"state dict mismatch: missing {missing}, unexpected {unexpected}")
    return m.eval()


def install():
    """-> the reference ``compute_fitness`` module, importable and CPU-bound."""
    if "compute_fitness_progen2" in sys.modules:
        return sys.modules["compute_fitness_progen2"]
    import torch
    torch.nn.Module.cuda = lambda self, *a, **k: self
    orig_to = torch.Tensor.to

    def to(self, *args, **kwargs):
        if args and str(args[0]).startswith("cuda"):
            return self
        return orig_to(self, *args, **kwargs)
    torch.Tensor.to = to
    _model_module()
    spec = importlib.util.spec_from_file_location("compute_fitness_progen2", os.path.join(REF, "compute_fitness.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules["compute_fitness_progen2"] = mod
    spec.loader.exec_module(mod)
    mod.create_model = lambda ckpt, fp16: load_model(ckpt)
    return mod
