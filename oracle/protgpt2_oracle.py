"""ORACLE — plain-torch GPT-2 forward (ProtGPT2) in fp32 / fp64 and its per-token log-probabilities, restating transformers'
models/gpt2/modeling_gpt2.py: GPT2Model.forward (inputs_embeds + position_embeds, the blocks, ln_f), GPT2Block.forward (pre-LN attention
and MLP with residuals), GPT2Attention (c_attn split into q / k / v, scaled dot product with a causal mask, c_proj), GPT2MLP (c_fc,
gelu_new, c_proj; Conv1D computes x @ W + b with W [in, out]), and GPT2LMHeadModel (lm_head tied to wte, no bias). Used by the GPU tests
as the fp64 yardstick."""
from __future__ import annotations

import math

import torch


def _w(st, k, dtype):
    t = st.get("transformer." + k, st.get(k))
    return t.to(dtype)


def gelu_new(x):
    """activations.py NewGELUActivation: 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3)))."""
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))


def logprob_rows(st: dict, ids, heads: int, dtype=torch.float64) -> torch.Tensor:
    """log_softmax of the logits of every position of one token row -> [T, vocab] (GPT2LMHeadModel.forward without labels)."""
    ids = torch.as_tensor(ids, dtype=torch.long)
    T = ids.numel()
    wte = _w(st, "wte.weight", dtype)
    x = wte[ids] + _w(st, "wpe.weight", dtype)[:T]
    d = x.shape[1]
    hd = d // heads
    mask = torch.ones((T, T), dtype=torch.bool).tril()
    n_layers = sum(1 for k in st if k.endswith("ln_1.weight"))
    ln = lambda v, p: torch.nn.functional.layer_norm(v, (d,), _w(st, p + ".weight", dtype), _w(st, p + ".bias", dtype), 1e-5)  # noqa: E731
    for i in range(n_layers):
        p = f"h.{i}."
        h = ln(x, p + "ln_1")
        qkv = h @ _w(st, p + "attn.c_attn.weight", dtype) + _w(st, p + "attn.c_attn.bias", dtype)
        q, k, v = (t.view(T, heads, hd).transpose(0, 1) for t in qkv.split(d, dim=1))
        s = (q @ k.transpose(1, 2)) / math.sqrt(hd)
        s = s.masked_fill(~mask, float("-inf"))
        o = (torch.softmax(s, dim=-1) @ v).transpose(0, 1).reshape(T, d)
        x = x + o @ _w(st, p + "attn.c_proj.weight", dtype) + _w(st, p + "attn.c_proj.bias", dtype)
        h = ln(x, p + "ln_2")
        m = gelu_new(h @ _w(st, p + "mlp.c_fc.weight", dtype) + _w(st, p + "mlp.c_fc.bias", dtype))
        x = x + m @ _w(st, p + "mlp.c_proj.weight", dtype) + _w(st, p + "mlp.c_proj.bias", dtype)
    x = ln(x, "ln_f")
    return torch.log_softmax(x @ wte.T, dim=-1)


def token_logprobs(st: dict, ids, heads: int, dtype=torch.float64) -> torch.Tensor:
    """log p(ids[t+1] | ids[<=t]) for t < T-1 -> [T-1]."""
    rows = logprob_rows(st, ids, heads, dtype)
    tgt = torch.as_tensor(ids[1:], dtype=torch.long)
    return rows[torch.arange(len(ids) - 1), tgt]
