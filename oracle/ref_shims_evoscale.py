"""ORACLE SUPPORT — TEST INFRASTRUCTURE ONLY (build container only: needs /root/reference).

Import shims that let the UNMODIFIED evoscale ``compute_fitness.py`` (proteingym/baselines/evoscale) run ESM C on the CPU:
  * stub packages for the structure / cloud / compression dependencies ESM C never calls (Bio, biotite, zstd, brotli, msgpack,
    msgpack_numpy, cloudpathlib, tenacity): any name imported from them is an inert placeholder class;
  * ``flash_attn`` blocked, so ``ESMC`` takes its SDPA path (the installed flash_attn's Triton rotary needs a CUDA device);
  * ``INFRA_PROVIDER=1`` so ``data_root`` is the working directory and the weights load from ``data/weights/...pth``;
  * ``Module.to("cuda")`` a no-op (the script moves the model to the GPU).
Nothing is copied from the reference."""
from __future__ import annotations

import importlib.abc
import importlib.machinery
import os
import sys
import types

REF = os.path.join(os.environ.get("PG_REFERENCE_ROOT", "/root/reference"), "proteingym", "baselines", "evoscale")
STUBS = ("Bio", "biotite", "zstd", "brotli", "msgpack", "msgpack_numpy", "cloudpathlib", "tenacity")
BLOCKED = ("flash_attn",)


def available() -> bool:
    return os.path.isfile(os.path.join(REF, "compute_fitness.py"))


class _Placeholder:
    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        return self


class _StubModule(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        v = type(name, (_Placeholder,), {})
        setattr(self, name, v)
        return v


class _Finder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    def find_spec(self, fullname, path=None, target=None):
        root = fullname.split(".")[0]
        if root in BLOCKED:
            raise ImportError(f"{fullname} is blocked for the CPU golden run")
        if root in STUBS:
            return importlib.machinery.ModuleSpec(fullname, self, is_package=True)
        return None

    def create_module(self, spec):
        m = _StubModule(spec.name)
        m.__path__ = []
        return m

    def exec_module(self, module):
        pass


def install():
    """-> the reference ``compute_fitness`` module, importable and CPU-bound."""
    if "compute_fitness_evoscale" in sys.modules:
        return sys.modules["compute_fitness_evoscale"]
    for name in list(sys.modules):
        if name.split(".")[0] in BLOCKED:
            del sys.modules[name]
    sys.meta_path.insert(0, _Finder())
    os.environ["INFRA_PROVIDER"] = "1"
    import torch
    orig_to = torch.nn.Module.to

    def to(self, *args, **kwargs):
        if args and str(args[0]).startswith("cuda"):
            return self
        return orig_to(self, *args, **kwargs)
    torch.nn.Module.to = to
    if REF not in sys.path:
        sys.path.insert(0, REF)
    import importlib.util
    spec = importlib.util.spec_from_file_location("compute_fitness_evoscale", os.path.join(REF, "compute_fitness.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules["compute_fitness_evoscale"] = mod
    spec.loader.exec_module(mod)
    return mod
