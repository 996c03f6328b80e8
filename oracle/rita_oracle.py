"""ORACLE — plain-torch restatement of the RITA reference (proteingym/baselines/rita), fp32 or fp64 on the CPU. Independent of the CUDA
library; used by the CPU tests (against the goldens of the unmodified reference) and by the GPU tests (fp64 per-token bounds).

  model        rita_modeling.py:244-252 (embedding, layers, final_norm), lm_head :285,:323
  layer        rita_modeling.py:197-210 (pre-LN attention and MLP blocks, residuals)
  attention    rita_modeling.py:136-176 (separate q/k/v with bias, rotary :39-67 over the full head, /sqrt(head_dim), causal -inf, softmax)
  RITA_gelu    rita_modeling.py:24-26
  calc_fitness compute_fitness.py:13-42 (chunks of 1023, both directions, mean target log-prob per chunk and direction, summed)
"""
from __future__ import annotations

import math

import numpy as np
import torch


def rita_gelu(x):
    return x * 0.5 * (1.0 + torch.tanh(0.79788456 * x * (1 + 0.044715 * x * x)))


def _ln(x, st, p):
    return torch.nn.functional.layer_norm(x, (x.shape[-1],), st[p + ".weight"], st[p + ".bias"], 1e-5)


def logprob_rows(st: dict, ids, heads: int, dtype=torch.float64, tied: bool = True) -> torch.Tensor:
    """log_softmax of the logits of every input position of one token row ``ids`` (the model input, ids[:-1] in calc_fitness) -> [T, vocab].
    ``st``: RITAModelForCausalLM state dict (``transformer.`` keys); ``tied``: the head is the embedding matrix, else lm_head.weight."""
    S = {k: v.to(dtype) for k, v in st.items()}
    ids = torch.as_tensor(ids, dtype=torch.long)
    T = ids.shape[0]
    x = S["transformer.embedding.weight"][ids]
    d = x.shape[-1]
    hd = d // heads
    causal = torch.triu(torch.ones(T, T, dtype=torch.bool), 1)
    L = 1 + max(int(k.split(".")[2]) for k in S if k.startswith("transformer.layers."))
    for i in range(L):
        p = f"transformer.layers.{i}."
        a = p + "self_attention."
        y = _ln(x, S, p + "attn_norm")
        q, k, v = (torch.nn.functional.linear(y, S[a + n + ".weight"], S[a + n + ".bias"]).view(T, heads, hd).transpose(0, 1)
                   for n in ("query", "key", "value"))
        inv = st[a + "rotary_embedding.inv_freq"].float()  # the reference builds its tables in fp32 (:59-63)
        freqs = torch.einsum("i,j->ij", torch.arange(T).type_as(inv), inv)
        emb = torch.cat((freqs, freqs), dim=-1)
        cos, sin = emb.cos().to(dtype), emb.sin().to(dtype)

        def rot(t):
            return torch.cat((-t[..., hd // 2:], t[..., :hd // 2]), dim=-1)
        q, k = q * cos + rot(q) * sin, k * cos + rot(k) * sin
        att = (q @ k.transpose(-2, -1)) * (1.0 / math.sqrt(hd))
        att = att.masked_fill(causal, float("-inf")).softmax(-1)
        o = (att @ v).transpose(0, 1).reshape(T, d)
        x = x + torch.nn.functional.linear(o, S[a + "proj.weight"], S[a + "proj.bias"])
        y = _ln(x, S, p + "mlp_norm")
        y = torch.nn.functional.linear(rita_gelu(torch.nn.functional.linear(y, S[p + "mlp.0.weight"], S[p + "mlp.0.bias"])),
                                       S[p + "mlp.2.weight"], S[p + "mlp.2.bias"])
        x = x + y
    x = _ln(x, S, "transformer.final_norm")
    head = S["transformer.embedding.weight"] if tied else S["lm_head.weight"]
    return torch.log_softmax(x @ head.T, dim=-1)


def mean_target_logprob(st, ids, heads, dtype=torch.float32, tied=True) -> float:
    """-CrossEntropyLoss()(logits(ids[:-1]), ids[1:]) of calc_fitness (:33-39); NaN when there is no target."""
    ids = list(ids)
    if len(ids) < 2:
        return math.nan
    lp = logprob_rows(st, ids[:-1], heads, dtype, tied)
    return float(lp[torch.arange(len(ids) - 1), torch.as_tensor(ids[1:])].mean())


def calc_fitness(st, prots, encode, heads, dtype=torch.float32, tied=True, context=1023) -> np.ndarray:
    """compute_fitness.py:13-42 restated: per protein, the sum over chunks and both directions of the mean target log-probability."""
    out = []
    for prot in prots:
        if len(prot) < context:
            chunks = [prot]
        else:
            chunks = [prot[i * context:(i + 1) * context] for i in range(1 + int(len(prot) / context))]
        total = 0.0
        for c in chunks:
            for p in (c, c[::-1]):
                total += mean_target_logprob(st, encode(p), heads, dtype, tied)
        out.append(total)
    return np.array(out, dtype=np.float64)
