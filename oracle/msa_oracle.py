"""ORACLE — TEST INFRASTRUCTURE ONLY. Not part of the product path.

CPU restatement (plain torch tensor ops, fp32 or fp64, no nn.Module) of ProteinGym's MSA Transformer masked-marginal path
(SURVEY.md §8 f3). Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py`` may import it; ``proteingym_b200`` never does.

Parity status: PINNED against the reference itself — ``oracle/gen_golden_msa_transformer.py`` runs the UNMODIFIED reference
(``compute_fitness.py::main --model_type MSA_transformer`` and the vendored ``MSATransformer``) on seeded synthetic checkpoints and
alignments and commits its outputs under ``tests/golden/msa_transformer_*``; ``tests/test_oracle_vs_golden.py`` checks this
restatement against them.

Every function cites the reference lines it restates (paths relative to /root/reference/proteingym/baselines/esm).
"""
from __future__ import annotations

import math

import torch

from .esm_oracle import MASK_IDX, TOK, gelu, layer_norm

CLS_IDX = 0


def tokenize_alignment(rows) -> torch.Tensor:
    """esm/data.py:300-336 (MSABatchConverter, one alignment; prepend_bos, no eos): rows = [(name, aligned string)] -> [R, L + 1]."""
    L = len(rows[0][1])
    if any(len(s) != L for _, s in rows):
        raise RuntimeError("Received unaligned sequences for input to MSA, all sequence lengths must be equal.")
    return torch.tensor([[CLS_IDX] + [TOK[c] for c in s] for _, s in rows], dtype=torch.int64)


def _lin(x, st, name):
    return x @ st[name + ".weight"].T + st[name + ".bias"]


# Emulated kernel faults, for measuring how far a test bound is from a real bug: each rounds one operand of the otherwise exact model
# to fp16 (the hi plane alone, as if a kernel dropped the lo plane). None (the default) is the model itself.
FAULTS = ("tied_qkv_f16", "tied_p_f16", "col_qkv_f16")


def _f16(t):
    return t.to(torch.float16).to(t.dtype)


def row_attention(x, st, p, heads, fault=None):
    """RowSelfAttention (axial_attention.py:78-200): tied attention — one [C, C] map per head, logits summed over the alignment rows,
    q scaled by head_dim^-0.5 / sqrt(R) (:78-80,125). The reference's row-batched path (:82-113) adds the same terms in row chunks."""
    R, C, B, d = x.shape
    hd = d // heads
    q = _lin(x, st, p + "q_proj").view(R, C, B, heads, hd)
    k = _lin(x, st, p + "k_proj").view(R, C, B, heads, hd)
    v = _lin(x, st, p + "v_proj").view(R, C, B, heads, hd)
    if fault == "tied_qkv_f16":  # the kernels' q carries head_dim^-0.5 (folded into the weights); 1/sqrt(R) is the softmax's
        q, k, v = _f16(q * hd ** -0.5) / math.sqrt(R), _f16(k), _f16(v)
    else:
        q = q * (hd ** -0.5 / math.sqrt(R))
    w = torch.einsum("rinhd,rjnhd->hnij", q, k).softmax(-1)
    if fault == "tied_p_f16":
        w = _f16(w)
    ctx = torch.einsum("hnij,rjnhd->rinhd", w, v).reshape(R, C, B, d)
    return _lin(ctx, st, p + "out_proj")


def column_attention(x, st, p, heads, fault=None):
    """ColumnSelfAttention (axial_attention.py:254-297): per column, attention over the R rows; a single row is v -> out_proj."""
    R, C, B, d = x.shape
    hd = d // heads
    if R == 1:
        return _lin(_lin(x, st, p + "v_proj"), st, p + "out_proj")
    q = _lin(x, st, p + "q_proj").view(R, C, B, heads, hd) * hd ** -0.5
    k = _lin(x, st, p + "k_proj").view(R, C, B, heads, hd)
    v = _lin(x, st, p + "v_proj").view(R, C, B, heads, hd)
    if fault == "col_qkv_f16":
        q, k, v = _f16(q), _f16(k), _f16(v)
    w = torch.einsum("icnhd,jcnhd->hcnij", q, k).softmax(-1)
    ctx = torch.einsum("hcnij,jcnhd->icnhd", w, v).reshape(R, C, B, d)
    return _lin(ctx, st, p + "out_proj")


def msa_forward(st: dict, tokens: torch.Tensor, layers: int, heads: int, dtype=torch.float32, fault=None) -> torch.Tensor:
    """MSATransformer.forward (model/msa_transformer.py:150-222) in eval mode, no padding: tokens [B, R, C] -> logits [B, R, C, V].
    ``fault``: one of FAULTS, applied in every layer."""
    if fault is not None and fault not in FAULTS:
        raise ValueError(f"unknown fault {fault!r}")
    st = {k: v.to(dtype) for k, v in st.items()}
    B, R, C = tokens.shape
    x = st["embed_tokens.weight"][tokens]
    # LearnedPositionalEmbedding (modules.py:254-271): positions = cumsum(non-pad) + padding_idx = column + 2
    x = x + st["embed_positions.weight"][torch.arange(C) + 2][None, None]
    if "msa_position_embedding" in st:
        if R > 1024:
            raise RuntimeError("MSA position embedding covers 1024 rows")
        x = x + st["msa_position_embedding"][:, :R]
    x = layer_norm(x, st["emb_layer_norm_before.weight"], st["emb_layer_norm_before.bias"])
    x = x.permute(1, 2, 0, 3)  # R, C, B, D
    for i in range(layers):
        # AxialTransformerLayer (modules.py:205-235): three pre-LN residual blocks (NormalizedResidualBlock, :390-406)
        p = f"layers.{i}.row_self_attention."
        x = x + row_attention(layer_norm(x, st[p + "layer_norm.weight"], st[p + "layer_norm.bias"]), st, p + "layer.", heads, fault)
        p = f"layers.{i}.column_self_attention."
        x = x + column_attention(layer_norm(x, st[p + "layer_norm.weight"], st[p + "layer_norm.bias"]), st, p + "layer.", heads, fault)
        p = f"layers.{i}.feed_forward_layer."
        h = layer_norm(x, st[p + "layer_norm.weight"], st[p + "layer_norm.bias"])
        x = x + _lin(gelu(_lin(h, st, p + "layer.fc1")), st, p + "layer.fc2")  # FeedForwardNetwork (modules.py:428-432)
    x = layer_norm(x, st["emb_layer_norm_after.weight"], st["emb_layer_norm_after.bias"]).permute(2, 0, 1, 3)
    # RobertaLMHead (modules.py:300-316), output matrix tied to embed_tokens
    h = gelu(_lin(x, st, "lm_head.dense"))
    h = layer_norm(h, st["lm_head.layer_norm.weight"], st["lm_head.layer_norm.bias"])
    return h @ st["embed_tokens.weight"].T + st["lm_head.bias"]


def optimal_window(i: int, seq_len_wo_special: int, model_window: int = 1024):
    """proteingym/utils/scoring_utils.py:43-52."""
    half = model_window // 2
    if seq_len_wo_special <= model_window:
        return 0, seq_len_wo_special
    if i < half:
        return 0, model_window
    if i >= seq_len_wo_special - half:
        return seq_len_wo_special - model_window, seq_len_wo_special
    return max(0, i - half), min(seq_len_wo_special, i + half)


def masked_marginal_table(st: dict, tokens: torch.Tensor, layers: int, heads: int, positions=None, dtype=torch.float32,
                          fault=None) -> torch.Tensor:
    """compute_fitness.py:383-399: for each column i (BOS included) mask (row 0, column i), forward the whole alignment (the
    1024-column optimal window around i when the alignment is longer) and keep log_softmax(logits)[row 0, column i].
    tokens [R, C] -> [len(positions), V] (positions default: every column)."""
    R, C = tokens.shape
    out = []
    for i in (range(C) if positions is None else positions):
        t = tokens.clone()
        t[0, i] = MASK_IDX
        start = 0
        if C > 1024:
            start, end = optimal_window(i, C + 1, 1024)  # the reference passes len(sequence) + 2 = C + 1 (:389)
            t = t[:, start:end]
        logits = msa_forward(st, t[None], layers, heads, dtype, fault)
        out.append(torch.log_softmax(logits[0, 0, i - start], dim=-1))
    return torch.stack(out)
