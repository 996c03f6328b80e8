"""ORACLE — TEST INFRASTRUCTURE ONLY. Not part of the product path.

CPU restatement (plain torch tensor ops, fp32 or fp64, no nn.Module) of ProteinGym's ESM C masked-marginal scoring
(``proteingym/baselines/evoscale``). Only ``tests/`` and the golden / bench scripts import it; ``proteingym_b200`` never does.
``oracle/gen_golden_esmc.py`` runs the unmodified reference on the CPU and commits its outputs under ``tests/golden/esmc_*``;
``tests/test_esmc_cpu.py`` checks this restatement against them.

Every function cites the reference lines it restates (paths relative to proteingym/baselines/evoscale).
"""
from __future__ import annotations

import math
import re

import numpy as np
import torch

CLS_IDX, PAD_IDX, EOS_IDX, MASK_IDX = 0, 1, 2, 32
# esm/utils/constants/esm3.py:52-58 (SEQUENCE_VOCAB)
VOCAB = ["<cls>", "<pad>", "<eos>", "<unk>", "L", "A", "G", "V", "S", "E", "R", "T", "I", "D", "P", "K", "Q", "N", "F", "Y", "M", "H",
         "W", "C", "X", "B", "U", "Z", "O", ".", "-", "|", "<mask>"]
TOK = {t: i for i, t in enumerate(VOCAB)}
AA20 = set("ACDEFGHIKLMNPQRSTVWY")


def tokenize(seq: str) -> torch.Tensor:
    """esm/utils/encoding.py tokenize_sequence with add_special_tokens: ``<cls> seq <eos>``."""
    return torch.tensor([CLS_IDX] + [TOK[c] for c in seq] + [EOS_IDX], dtype=torch.int64)


def layer_norm(x, w, b=None, eps=1e-5):
    """torch.nn.LayerNorm (biased variance, eps 1e-5); ``b`` None for the bias-free norms (q_ln, k_ln, transformer.norm)."""
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    y = (x - mu) / torch.sqrt(var + eps) * w
    return y if b is None else y + b


def rotary_tables(T, dtype):
    """esm/layers/rotary.py:136-165: inv_freq = 1/10000^(arange(0, 64, 2)/64) and torch.outer(t, inv_freq), both fp32."""
    inv_freq = 1.0 / (10000 ** (torch.arange(0, 64, 2, dtype=torch.float32) / 64))
    freqs = torch.outer(torch.arange(T, dtype=torch.float32), inv_freq)
    return freqs.cos().to(dtype), freqs.sin().to(dtype)


def apply_rotary(x, cos, sin):
    """esm/layers/rotary.py:36-65 (interleaved=False): x [B, T, H, 64]; x*cos + rotate_half(x)*sin with the tables repeated twice."""
    c = torch.cat((cos, cos), -1)[None, :, None, :]
    s = torch.cat((sin, sin), -1)[None, :, None, :]
    x1, x2 = x.chunk(2, dim=-1)
    return x * c + torch.cat((-x2, x1), -1) * s


def esmc_forward(st: dict, tokens: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    """Logits [B, T, 64]. ESMC.forward (esm/models/esmc.py:117-173) on the SDPA path with an all-True mask (no padding):
    TransformerStack (esm/layers/transformer_stack.py:42-94), UnifiedTransformerBlock (esm/layers/blocks.py:122-162),
    MultiHeadAttention (esm/layers/attention.py:19-85), SwiGLU FFN (blocks.py:15-43), RegressionHead (esm/layers/regression_head.py)."""
    W = lambda n: st[n].to(dtype)
    B, T = tokens.shape
    d = st["embed.weight"].shape[1]
    H = d // 64
    layers = 1 + max(int(k.split(".")[2]) for k in st if k.startswith("transformer.blocks."))
    scale = math.sqrt(layers / 36)  # transformer_stack.py:48-50
    x = W("embed.weight")[tokens]
    cos, sin = rotary_tables(T, dtype)
    for i in range(layers):
        p = f"transformer.blocks.{i}."
        h = layer_norm(x, W(p + "attn.layernorm_qkv.0.weight"), W(p + "attn.layernorm_qkv.0.bias"))
        q, k, v = (h @ W(p + "attn.layernorm_qkv.1.weight").T).chunk(3, dim=-1)
        q = layer_norm(q, W(p + "attn.q_ln.weight"))
        k = layer_norm(k, W(p + "attn.k_ln.weight"))
        q = apply_rotary(q.view(B, T, H, 64), cos, sin).transpose(1, 2)
        k = apply_rotary(k.view(B, T, H, 64), cos, sin).transpose(1, 2)
        v = v.view(B, T, H, 64).transpose(1, 2)
        a = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(64), dim=-1)  # F.scaled_dot_product_attention
        ctx = (a @ v).transpose(1, 2).reshape(B, T, d)
        x = x + (ctx @ W(p + "attn.out_proj.weight").T) / scale
        h = layer_norm(x, W(p + "ffn.0.weight"), W(p + "ffn.0.bias"))
        g, u = (h @ W(p + "ffn.1.weight").T).chunk(2, dim=-1)
        x = x + ((g * torch.sigmoid(g) * u) @ W(p + "ffn.3.weight").T) / scale
    x = layer_norm(x, W("transformer.norm.weight"))
    h = x @ W("sequence_head.0.weight").T + W("sequence_head.0.bias")
    h = h * 0.5 * (1.0 + torch.erf(h / math.sqrt(2.0)))
    h = layer_norm(h, W("sequence_head.2.weight"), W("sequence_head.2.bias"))
    return h @ W("sequence_head.3.weight").T + W("sequence_head.3.bias")


def window(seq_pos: int, seq_len: int, window_size: int = 1024):
    """compute_fitness.py:346-375 -> (start, end) residue slice of the window holding 0-based residue seq_pos (whole sequence when
    seq_len <= window_size - 2)."""
    if seq_len <= window_size - 2:
        return 0, seq_len
    half = (window_size - 2) // 2
    start = max(0, seq_pos - half)
    end = min(seq_len, start + window_size - 2)
    if end == seq_len:
        start = max(0, seq_len - (window_size - 2))
    return start, end


def masked_rows(st, seq: str, seq_positions, dtype=torch.float32, batch=8) -> torch.Tensor:
    """compute_fitness.py:359-425: for each 0-based residue p, mask its token in ``<cls> window <eos>`` and keep
    log_softmax(logits)[token]. -> [P, 64]."""
    out = torch.empty((len(seq_positions), 64), dtype=dtype)
    groups = {}
    for r, p in enumerate(seq_positions):
        groups.setdefault(window(p, len(seq)), []).append((r, p))
    for (start, end), members in groups.items():
        toks = tokenize(seq[start:end])
        for c in range(0, len(members), batch):
            chunk = members[c:c + batch]
            tb = toks.unsqueeze(0).repeat(len(chunk), 1)
            for j, (_, p) in enumerate(chunk):
                tb[j, p - start + 1] = MASK_IDX
            lp = torch.log_softmax(esmc_forward(st, tb, dtype), dim=-1)
            for j, (r, p) in enumerate(chunk):
                out[r] = lp[j, p - start + 1]
    return out


def parse(mutant: str, seq: str):
    """compute_fitness.py:69-136: [(seq_pos, wt, mt)] or None when the reference skips the mutant."""
    sites = []
    for sub in mutant.split(":"):
        m = re.match(r"([A-Z])(\d+)([A-Z])", sub)
        if not m:
            return None
        wt, pos, mt = m.group(1), int(m.group(2)) - 1, m.group(3)
        if pos < 0 or pos >= len(seq) or seq[pos] != wt:
            return None
        sites.append((pos, wt, mt))
    return sites


def score_mutants(mutants, seq: str, rows_by_pos: dict) -> np.ndarray:
    """compute_fitness.py:427-474, 592: sum over sites of log_softmax[mt] - log_softmax[wt]; NaN for skipped mutants.
    ``rows_by_pos``: 0-based residue -> [64] log-probs."""
    out = []
    for m in mutants:
        sites = parse(str(m), seq)
        if sites is None:
            out.append(np.nan)
            continue
        out.append(sum(float(rows_by_pos[p][TOK[mt]] - rows_by_pos[p][TOK[wt]]) for p, wt, mt in sites))
    return np.array(out, dtype=np.float64)


def score_assay(st, seq: str, mutants, dtype=torch.float32):
    """Scores of the whole assay (only the residues some valid mutant uses are run, compute_fitness.py:335-342)."""
    pos = sorted({p for m in mutants for p, _, _ in (parse(str(m), seq) or [])})
    rows = masked_rows(st, seq, pos, dtype) if pos else torch.empty(0, 64)
    return score_mutants(mutants, seq, {p: rows[i] for i, p in enumerate(pos)})
