"""ORACLE — plain-torch restatement of the ProGen3 scorer (proteingym/baselines/progen3/progen3/) in fp64 (or fp32), on the canonical
state of include/pgscore.h's PG_ARCH_PROGEN3 (checkpoint.normalise_progen3_state). It cites the reference lines it restates:

  embedding          modeling.py:374,441      x = embed_tokens[ids] + embed_seq_id[0]
  RMSNorm            modeling.py:168-190      x * rsqrt(mean(x^2) + eps) * w (flash-attn rms_norm_fn)
  attention          model/attention.py:38-91, 217-249: q/k/v without bias, kv_heads key/value heads (repeat_kv), rotate-half rotary over
                     the whole head (inv_freq = theta^-(2i/hd), tables cat(angles, angles)), causal softmax(q k^T / sqrt(hd)) v, o_proj
  MoE                model/moe.py:62-134      softmax(gate x) in fp32, topk, renormalise, experts SiLU MLP or GLU, weighted, index_add_ in
                     expert order; one expert: its output alone
  head               modeling.py:495,600      final RMSNorm, lm_head without bias
  score              scorer.py:64-101         per direction mean log p over the targets, ll = (fwd + rev) / 2

``routing`` overrides the router: a list over layers of (experts [T, k] int, weights [T, k]) arrays, used instead of the computed ones
(the kernel's own routing, to separate arithmetic error from routing decisions)."""
from __future__ import annotations

import numpy as np
import torch


def rms(x, w, eps):
    return x * torch.rsqrt((x * x).mean(-1, keepdim=True) + eps) * w


def rotate_half(x):
    h = x.shape[-1] // 2
    return torch.cat((-x[..., h:], x[..., :h]), dim=-1)


def forward(state: dict, conf, ids, dtype=torch.float64, routing=None):
    """-> (log-probabilities [T, vocab] of the next token after each row, routes): routes[l] = (experts [T, k], weights [T, k], probs [T, E])
    as the router chose them (or as ``routing`` imposed them; probs are the router's own either way)."""
    S = {k: v.to(dtype) for k, v in state.items()}
    ids = torch.as_tensor(ids, dtype=torch.long)
    T, d, H, Hk = len(ids), conf.embed_dim, conf.heads, conf.kv_heads
    hd, E, K, eps = d // H, conf.n_experts, conf.top_k, conf.rms_eps
    x = S["embed_tokens.weight"][ids] + S["embed_seq_id.weight"][0]
    inv = conf.rope_theta ** -(torch.arange(0, hd, 2, dtype=dtype) / hd)
    ang = torch.outer(torch.arange(T, dtype=dtype), inv)
    ang = torch.cat((ang, ang), dim=1)
    cos, sin = ang.cos()[:, None, :], ang.sin()[:, None, :]
    mask = torch.ones(T, T, dtype=torch.bool).tril()
    routes = []
    for l in range(conf.layers):
        p = f"layers.{l}."
        h = rms(x, S[p + "input_layernorm.weight"], eps)
        q = (h @ S[p + "self_attn.q_proj.weight"].T).view(T, H, hd)
        k = (h @ S[p + "self_attn.k_proj.weight"].T).view(T, Hk, hd)
        v = (h @ S[p + "self_attn.v_proj.weight"].T).view(T, Hk, hd)
        q, k = q * cos + rotate_half(q) * sin, k * cos + rotate_half(k) * sin
        k, v = k.repeat_interleave(H // Hk, dim=1), v.repeat_interleave(H // Hk, dim=1)
        s = torch.einsum("thd,shd->hts", q, k) / np.sqrt(hd)
        a = torch.softmax(s.masked_fill(~mask, float("-inf")), dim=-1)
        o = torch.einsum("hts,shd->thd", a, v).reshape(T, d)
        x = x + o @ S[p + "self_attn.o_proj.weight"].T
        h = rms(x, S[p + "post_attention_layernorm.weight"], eps)
        m = p + "block_sparse_moe."
        w1 = S[m + "w1"].view(E, -1, d)
        w3 = S[m + "w3"].view(E, -1, d) if conf.gated_mlp else None
        w2 = S[m + "w2"].view(E, d, -1)
        if E == 1:
            probs = torch.ones(T, 1, dtype=dtype)
            ex, wt = torch.zeros(T, 1, dtype=torch.long), torch.ones(T, 1, dtype=dtype)
        else:
            probs = torch.softmax(h @ S[m + "gate.weight"].T, dim=-1)
            wt, ex = torch.topk(probs, K, dim=-1)  # ties: see include/pgscore.h (lower expert index first)
            wt = wt / wt.sum(-1, keepdim=True)
        if routing is not None:
            ex = torch.as_tensor(np.asarray(routing[l][0]), dtype=torch.long)
            wt = torch.as_tensor(np.asarray(routing[l][1]), dtype=dtype)
        routes.append((ex.numpy().copy(), wt.numpy().copy(), probs.numpy().copy()))
        out = torch.zeros_like(h)
        for e in range(E):
            tok, slot = torch.where(ex == e)
            if len(tok) == 0:
                continue
            z = h[tok] @ w1[e].T
            z = z * torch.sigmoid(z)
            if w3 is not None:
                z = z * (h[tok] @ w3[e].T)
            out.index_add_(0, tok, (z @ w2[e].T) * wt[tok, slot, None])
        x = x + out
    logits = rms(x, S["norm.weight"], eps) @ S["lm_head.weight"].T
    return torch.log_softmax(logits, dim=-1), routes


def token_logp(state, conf, ids, dtype=torch.float64, routing=None):
    """log p(ids[t+1] | ids[<=t]) for t < T-1 (numpy), and the routes."""
    lp, routes = forward(state, conf, ids, dtype, routing)
    ids = np.asarray(ids)
    return lp[np.arange(len(ids) - 1), ids[1:]].numpy(), routes


def score(state, conf, seqs, dtype=torch.float64):
    """(log_likelihood, perplexity) per sequence as ProGen3Scorer.score_batch computes them (float64)."""
    from proteingym_b200.progen3_engine import Progen3Tokenizer
    tok = Progen3Tokenizer()
    ll = []
    for s in seqs:
        dirs = [token_logp(state, conf, tok.encode(s, rev), dtype)[0].mean() for rev in (False, True)]
        ll.append((dirs[0] + dirs[1]) / 2)
    ll = np.array(ll, dtype=np.float64)
    return ll, np.exp(-ll)


def topk_gaps(probs: np.ndarray, k: int) -> np.ndarray:
    """Per token: the gap between the k-th and (k+1)-th router probability (inf when k == E)."""
    if probs.shape[1] <= k:
        return np.full(probs.shape[0], np.inf)
    srt = -np.sort(-probs, axis=1)
    return srt[:, k - 1] - srt[:, k]
