"""ORACLE SUPPORT — TEST INFRASTRUCTURE ONLY (build container only: needs /root/reference).

Lets the UNMODIFIED ``proteingym/baselines/PoET/scripts/score.py`` run ``main()`` on the CPU:
  * ``flash_attn`` is hidden (``sys.modules["flash_attn"] = None``), so ``attention_flash.py`` takes its standard-attention branch;
  * ``FlashAttentionImpl.forward_standard_attn`` is replaced: the stock one pads the packed inputs, which the packed PoET inputs
    refuse (``to_paddedable=False``). The replacement runs softmax attention per ``cu_seqlens`` segment in the input dtype, with the
    causal mask aligned bottom-right as flash-attn's varlen kernels align it, over query chunks of at most 2048 rows (a 24 576-row
    segment would otherwise build a [heads, T, T] score tensor of tens of GB);
  * ``Module.cuda()`` / ``Tensor.cuda()`` are no-ops and ``Module.half()`` is the identity: the pin is the fp32 model;
  * ``pyzstd`` is a stub whose ``decompress`` returns its input (the fixtures are plain-text a3m files named ``*.a3m.zst``).
Nothing is copied from the reference."""
from __future__ import annotations

import importlib.util
import os
import sys
import types

REF = os.path.join(os.environ.get("PG_REFERENCE_ROOT", "/root/reference"), "proteingym", "baselines", "PoET")
Q_CHUNK = 2048


def available() -> bool:
    return os.path.isfile(os.path.join(REF, "scripts", "score.py"))


def _standard_attn(self, q, k, v, attn_mask=None, causal=False, need_weights=False):
    import copy

    import torch
    assert attn_mask is None and not need_weights
    scale = self.softmax_scale if self.softmax_scale is not None else q.x.size(-1) ** -0.5
    cq, ck = q.cu_seqlens_cpu.tolist(), k.cu_seqlens_cpu.tolist()
    out = torch.empty_like(q.x)
    for i in range(len(cq) - 1):
        q0, q1, k0, k1 = cq[i], cq[i + 1], ck[i], ck[i + 1]
        Lq, Lk = q1 - q0, k1 - k0
        kk = k.x[k0:k1].transpose(0, 1)  # [h, Lk, d]
        vv = v.x[k0:k1].transpose(0, 1)
        for a in range(0, Lq, Q_CHUNK):
            b = min(a + Q_CHUNK, Lq)
            qq = q.x[q0 + a:q0 + b].transpose(0, 1)  # [h, n, d]
            s = torch.matmul(qq, kk.transpose(1, 2)) * scale
            if causal:  # bottom-right: query row r sees keys <= r + Lk - Lq
                r = torch.arange(a, b).unsqueeze(1) + (Lk - Lq)
                s = s.masked_fill(torch.arange(Lk).unsqueeze(0) > r, float("-inf"))
            p = torch.softmax(s, dim=-1)
            out[q0 + a:q0 + b] = torch.matmul(p, vv).transpose(0, 1)
    o = copy.copy(q)
    o.x = out
    return o, None


def install():
    """-> the reference ``score`` module (scripts/score.py), importable and CPU-bound."""
    if "poet_score_ref" in sys.modules:
        return sys.modules["poet_score_ref"]
    import torch
    sys.modules["flash_attn"] = None
    if "pyzstd" not in sys.modules:
        stub = types.ModuleType("pyzstd")
        stub.decompress = lambda data: data
        sys.modules["pyzstd"] = stub
    torch.nn.Module.cuda = lambda self, *a, **k: self
    torch.nn.Module.half = lambda self, *a, **k: self
    torch.Tensor.cuda = lambda self, *a, **k: self
    if REF not in sys.path:
        sys.path.insert(0, REF)
    from poet.models.modules import attention_flash
    attention_flash.FlashAttentionImpl.forward_standard_attn = _standard_attn
    spec = importlib.util.spec_from_file_location("poet_score_ref", os.path.join(REF, "scripts", "score.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules["poet_score_ref"] = mod
    spec.loader.exec_module(mod)
    return mod
