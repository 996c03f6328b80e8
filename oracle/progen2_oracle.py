"""ORACLE — plain-torch restatement of the ProGen2 reference (proteingym/baselines/progen2), fp32 or fp64 on the CPU. Independent of the
CUDA library; used by the CPU tests (against the goldens of the unmodified reference) and by the GPU tests (fp64 per-token bounds).
Paths below are under proteingym/baselines/progen2/.

  model        models/progen/modeling_progen.py:389-401, 486-498 (wte, no position embedding, blocks, ln_f), lm_head with bias :541, :652
  block        modeling_progen.py:244-282 (h = ln_1(x); x = attn(h) + mlp(h) + x)
  attention    modeling_progen.py:146-214 (bias-free qkv_proj viewed as 8 shards of [q | v | k] :157-168; interleaved rotary on the first
               rotary_dim dims :178-194 with tables :38-57; q.k / sqrt(head_dim) in fp32, causal fill -1e9, softmax :113-135;
               bias-free out_proj)
  mlp          modeling_progen.py:224-241 (fc_in, gelu_new, fc_out, with biases)
  calc_fitness compute_fitness.py:34-86 (chunks of n_positions, both directions, terminal target dropped, CrossEntropy over logits
               5..29, summed, / 2, / len(prot))
"""
from __future__ import annotations

import math

import numpy as np
import torch

MP_NUM = 8  # modeling_progen.py:158


def gelu_new(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * torch.pow(x, 3.0))))


def _ln(x, S, p):
    return torch.nn.functional.layer_norm(x, (x.shape[-1],), S[p + ".weight"], S[p + ".bias"], 1e-5)


def rotary_tables(rotary_dim: int, T: int):
    """sin, cos [T, rotary_dim/2] in fp32 as fixed_pos_embedding builds them (modeling_progen.py:38-44)."""
    inv_freq = 1.0 / (10000 ** (torch.arange(0, rotary_dim, 2) / rotary_dim))
    sinusoid = torch.einsum("i , j -> i j", torch.arange(T), inv_freq).float()
    return torch.sin(sinusoid), torch.cos(sinusoid)


def _rotate(x, sin, cos):
    """apply_rotary_pos_emb (:53-57) on x [T, heads, r]: pairs (2i, 2i+1) rotated by angle i (rotate_every_two, :47-51)."""
    s, c = sin[:, None, :].repeat_interleave(2, -1), cos[:, None, :].repeat_interleave(2, -1)
    r = torch.stack((-x[..., 1::2], x[..., ::2]), dim=-1).flatten(-2)
    return x * c + r * s


def logits(st: dict, ids, heads: int, rotary_dim, dtype=torch.float64) -> torch.Tensor:
    """Logits [T, vocab] of every input position of one token row ``ids``. ``st``: ProGenForCausalLM state dict (``transformer.`` keys);
    ``rotary_dim`` None rotates the whole head (:187-190). The rotary tables are built in fp32 like the reference's, then cast."""
    S = {k: v.to(dtype) for k, v in st.items() if v.dtype.is_floating_point}
    ids = torch.as_tensor(ids, dtype=torch.long)
    T = ids.shape[0]
    x = S["transformer.wte.weight"][ids]
    d = x.shape[-1]
    hd = d // heads
    rd = hd if rotary_dim is None else rotary_dim
    sin, cos = (t.to(dtype) for t in rotary_tables(rd, T))
    causal = torch.tril(torch.ones(T, T, dtype=torch.bool))
    L = 1 + max(int(k.split(".")[2]) for k in S if k.startswith("transformer.h."))
    for i in range(L):
        p = f"transformer.h.{i}."
        h = _ln(x, S, p + "ln_1")
        qkv = (h @ S[p + "attn.qkv_proj.weight"].T).view(T, MP_NUM, -1)
        q, v, k = (t.reshape(T, heads, hd) for t in torch.split(qkv, d // MP_NUM, dim=-1))  # shard s holds heads s*heads/8 ..
        q = torch.cat([_rotate(q[..., :rd], sin, cos), q[..., rd:]], -1)
        k = torch.cat([_rotate(k[..., :rd], sin, cos), k[..., rd:]], -1)
        q, k, v = (t.transpose(0, 1) for t in (q, k, v))
        att = (q @ k.transpose(-1, -2)) / math.sqrt(hd)
        att = torch.where(causal, att, torch.tensor(-1e9, dtype=dtype)).softmax(-1)
        o = (att @ v).transpose(0, 1).reshape(T, d) @ S[p + "attn.out_proj.weight"].T
        m = torch.nn.functional.linear(gelu_new(torch.nn.functional.linear(h, S[p + "mlp.fc_in.weight"], S[p + "mlp.fc_in.bias"])),
                                       S[p + "mlp.fc_out.weight"], S[p + "mlp.fc_out.bias"])
        x = o + m + x
    x = _ln(x, S, "transformer.ln_f")
    return torch.nn.functional.linear(x, S["lm_head.weight"], S["lm_head.bias"])


def token_logprobs(st, ids, heads, rotary_dim, dtype=torch.float64) -> torch.Tensor:
    """log p(ids[t+1] | ids[<=t]) over the scored columns 5..29, t = 0 .. len-2 (the per-token terms of calc_fitness's mean)."""
    lg = logits(st, list(ids)[:-1], heads, rotary_dim, dtype)[:, 5:30]
    return torch.log_softmax(lg, -1)[torch.arange(len(ids) - 1), torch.as_tensor(list(ids)[1:]) - 5]


def chunk_loss(st, ids, heads, rotary_dim, dtype=torch.float32) -> float:
    """-CrossEntropyLoss of one (chunk, direction) (:55-78); NaN when no target remains; raises where the reference fails."""
    ids = list(ids)
    if len(ids) < 2:
        raise ValueError("fewer than two tokens")
    if ids[-1] in (3, 4):
        ids = ids[:-1]
    if any(t in (3, 4) for t in ids[1:]):
        raise AssertionError("terminal among the targets")
    if len(ids) < 2:
        return math.nan
    return float(token_logprobs(st, ids, heads, rotary_dim, dtype).mean())


def calc_fitness(st, prots, encode, heads, rotary_dim, context, dtype=torch.float32) -> np.ndarray:
    """compute_fitness.py:34-86 restated with reduction='mean'."""
    out = []
    for prot in prots:
        if len(prot) < context:
            chunks = [prot]
        else:
            chunks = [prot[i * context:(i + 1) * context] for i in range(1 + int(len(prot) / context))]
        total = 0.0
        for c in chunks:
            for p in (c, c[::-1]):
                total += chunk_loss(st, encode(p), heads, rotary_dim, dtype)
        out.append(total / 2.0 / len(prot))
    return np.array(out, dtype=np.float64)
