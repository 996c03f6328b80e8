"""ORACLE — TEST INFRASTRUCTURE ONLY. Not part of the product path.

CPU restatement (plain torch ops, fp32/fp64) of ProteinGym's Tranception autoregressive scorer:
model forward (tranception/model_pytorch.py:50-88 slopes + depthwise conv, :155-183 attention, :201-263, :265-360 blocks,
:438-632 model, :731-863 LM head + retrieval fusion) and the scoring arithmetic (tranception/utils/scoring_utils.py:16-31,
:47-60, :77-203; model_pytorch.py:878-938). Paths relative to /root/reference/proteingym/baselines/tranception.

Parity status: PINNED against a hybrid of the reference — ``TranceptionLMHeadModel`` cannot be constructed under
transformers 5.x (SURVEY.md §8c), so ``oracle/gen_golden_tranception.py`` runs the reference's own ``TranceptionBlock``
modules, ``get_slopes`` and the unmodified ``scoring_utils.get_sequence_slices`` / ``get_tranception_scores_mutated_sequences``
around a thin wrapper and commits the outputs to tests/golden/; tests/test_oracle_vs_golden.py checks this file against them.
"""
from __future__ import annotations

import math

import numpy as np
import pandas as pd
import torch

VOCAB = ["[UNK]", "[CLS]", "[SEP]", "[PAD]", "[MASK]"] + list("ACDEFGHIKLMNPQRSTVWY")
TOK = {t: i for i, t in enumerate(VOCAB)}
CLS, SEP, PAD = 1, 2, 3
AA_vocab = "ACDEFGHIKLMNPQRSTVWY"


def tokenize(seq: str) -> list:
    """Basic_tokenizer: single-character vocabulary, ``[CLS] seq [SEP]`` (utils/tokenizers/Basic_tokenizer)."""
    return [CLS] + [TOK.get(c, 0) for c in seq] + [SEP]


def get_slopes(n, mode="grouped_alibi"):
    """model_pytorch.py:50-71. grouped_alibi: slopes for n//4 heads, the list repeated 4x."""
    def pow2(n):
        start = 2 ** (-2 ** -(math.log2(n) - 3))
        return [start * start ** i for i in range(n)]
    if mode == "grouped_alibi":
        n = n // 4
    if math.log2(n).is_integer():
        res = pow2(n)
    else:
        c = 2 ** math.floor(math.log2(n))
        res = pow2(c) + get_slopes(2 * c, mode="standard_alibi")[0::2][:n - c]
    return res * 4 if mode == "grouped_alibi" else res


def layer_norm(x, w, b, eps):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * w + b


def depthwise_causal_conv(x, w, b, tile=0):
    """SpatialDepthWiseConvolution (model_pytorch.py:73-88): Conv1d(groups=hd, padding=k-1) then drop the last k-1 outputs
    => out[t] = b + sum_j w[:, j] * x[t - (k-1) + j]. x: [B, h, T, hd]; w: [hd, 1, k]; b: [hd].
    ``tile`` > 0 (emulated fault): a look-back term is dropped when its input row lies in an earlier tile of ``tile`` rows."""
    k = w.shape[-1]
    B, h, T, hd = x.shape
    xp = torch.cat([x.new_zeros(B, h, k - 1, hd), x], dim=2)
    out = x.new_zeros(B, h, T, hd) + b
    for j in range(k):
        term = xp[:, :, j:j + T, :] * w[:, 0, j]
        if tile:
            term = term * (torch.arange(T) % tile >= k - 1 - j).to(x.dtype)[:, None]
        out = out + term
    return out


# Emulated kernel faults, for measuring how far a test bound is from a real bug. None (the default) is the model itself.
#   attn_qkv_f16          the conv'd (q / sqrt(hd)), k, v rounded to fp16 before QK^T and PV (a dropped lo plane)
#   attn_p_f16            the softmax P rounded to fp16 before PV
#   conv_in_f16           the raw q / k / v rounded to fp16 before the depthwise conv
#   conv_tile_edge        conv look-back taps that cross a multiple of 64 rows dropped (a lost halo between conv tiles, or a
#                         wrong look-back pointer into the wild-type prefix)
#   alibi_slope_by_group  head h takes slopes[h // (heads / 4)], its conv group, instead of its own slope
FAULTS = ("attn_qkv_f16", "attn_p_f16", "conv_in_f16", "conv_tile_edge", "alibi_slope_by_group")


def _f16(t):
    return t.to(torch.float16).to(t.dtype)


def forward(st, ids, layers, heads, ln_eps=1e-5, dtype=torch.float32, rnd=None, fault=None):
    """logits [B, T, V] for right-padded ids [B, T] of EQUAL real length (callers group by length; padding never influences
    earlier positions under the causal mask, so per-length evaluation equals the reference's padded batches).
    ``fault``: one of FAULTS, applied in every layer."""
    if fault is not None and fault not in FAULTS:
        raise ValueError(f"unknown fault {fault!r}")
    rnd = rnd or (lambda t: t)
    W = lambda n: st[n].to(dtype)
    wte = W("transformer.wte.weight")
    B, T = ids.shape
    d = wte.shape[1]
    hd = d // heads
    g = heads // 4
    x = wte[ids]
    slopes = get_slopes(heads)
    if fault == "alibi_slope_by_group":
        slopes = [slopes[h // g] for h in range(heads)]
    slopes = torch.tensor(slopes, dtype=dtype)
    alibi = slopes[:, None, None] * torch.arange(T, dtype=dtype)[None, None, :]  # [h, 1, T]  (model_pytorch.py:376-380)
    causal = torch.tril(torch.ones(T, T, dtype=torch.bool))
    for i in range(layers):
        p = f"transformer.h.{i}."
        h_ = rnd(layer_norm(x, W(p + "ln_1.weight"), W(p + "ln_1.bias"), ln_eps))
        qkv = h_ @ rnd(W(p + "attn.c_attn.weight")) + W(p + "attn.c_attn.bias")  # Conv1D: x @ W[in,out] + b (:224)
        q, k, v = [t.view(B, T, heads, hd).permute(0, 2, 1, 3) for t in qkv.split(d, dim=2)]
        if fault == "conv_in_f16":
            q, k, v = _f16(q), _f16(k), _f16(v)
        tile = 64 if fault == "conv_tile_edge" else 0
        def conv_groups(t, nm):  # :240-251: heads [0,g) untouched; groups 1..3 get kernels 3,5,7
            parts = [t[:, :g]]
            for ki in range(3):
                parts.append(depthwise_causal_conv(t[:, (ki + 1) * g:(ki + 2) * g], W(p + f"attn.{nm}_depthwiseconv.{ki}.conv.weight"),
                                                   W(p + f"attn.{nm}_depthwiseconv.{ki}.conv.bias"), tile))
            return torch.cat(parts, dim=1)
        q, k, v = conv_groups(q, "query"), conv_groups(k, "key"), conv_groups(v, "value")
        q, k, v = rnd(q / float(hd) ** 0.5), rnd(k), rnd(v)  # (scale applied to q here; algebraically = :158-159)
        if fault == "attn_qkv_f16":
            q, k, v = _f16(q), _f16(k), _f16(v)
        s = q @ k.transpose(-1, -2)
        s = torch.where(causal, s, torch.tensor(-1e4, dtype=dtype))  # :162-165
        s = s + alibi[None]                                          # :167-168
        a = torch.softmax(s, dim=-1)
        if fault == "attn_p_f16":
            a = _f16(a)
        o = rnd((rnd(a) @ v).permute(0, 2, 1, 3).reshape(B, T, d))
        x = x + o @ rnd(W(p + "attn.c_proj.weight")) + W(p + "attn.c_proj.bias")
        h_ = rnd(layer_norm(x, W(p + "ln_2.weight"), W(p + "ln_2.bias"), ln_eps))
        h_ = torch.relu(h_ @ rnd(W(p + "mlp.c_fc.weight")) + W(p + "mlp.c_fc.bias"))
        h_ = rnd(h_ * h_)                                            # activations.py:79-84
        x = x + h_ @ rnd(W(p + "mlp.c_proj.weight")) + W(p + "mlp.c_proj.bias")
    x = layer_norm(x, W("transformer.ln_f.weight"), W("transformer.ln_f.bias"), ln_eps)
    return x @ W("lm_head.weight").T                                 # lm_head, no bias (:783)


def sequence_logprob(st, seq, layers, heads, ln_eps=1e-5, dtype=torch.float32, log_prior=None, alpha=0.0, start=0, end=None,
                     msa_start=0, msa_end=None, flip=False, rnd=None):
    """Sum over predicted tokens of log p(tok_{t+1} | tok_{<=t}) for ``[CLS] seq [SEP]`` (scoring_utils.py:121-128), with the
    optional retrieval fusion of model_pytorch.py:806-830 on the overlap of the slice [start, end) with [msa_start, msa_end)."""
    ids = torch.tensor([tokenize(seq)], dtype=torch.int64)
    lp = torch.log_softmax(forward(st, ids, layers, heads, ln_eps, dtype, rnd)[0, :-1], dim=-1)  # [T-1, V]
    if log_prior is not None:
        end = start + len(seq) if end is None else end
        msa_end = log_prior.shape[0] if msa_end is None else msa_end
        lo, hi = max(start, msa_start), min(end, msa_end)
        if hi > lo:
            sl = log_prior[lo:hi].to(dtype)
            if flip:
                sl = torch.flip(sl, dims=(0,))
                a0 = max(0, end - msa_end)
            else:
                a0 = max(0, msa_start - start)
            fused = lp.clone()
            fused[a0:a0 + (hi - lo)] = (1 - alpha) * lp[a0:a0 + (hi - lo)] + alpha * sl
            lp = fused
    labels = ids[0, 1:]
    return lp.gather(1, labels[:, None]).sum().item()


def logprob_rows(st, seqs, layers, heads, ln_eps=1e-5, dtype=torch.float64, fault=None):
    """Per string in ``seqs``: the log-softmax rows [len(s) + 1, V] (numpy) of every predicted position of ``[CLS] s [SEP]``
    (row t predicts token t + 1), unfused. ``fault``: one of FAULTS."""
    out = []
    with torch.no_grad():
        for s in seqs:
            ids = torch.tensor([tokenize(s)], dtype=torch.int64)
            out.append(torch.log_softmax(forward(st, ids, layers, heads, ln_eps, dtype, fault=fault)[0, :-1], dim=-1).numpy())
    return out


def fused_logprob_rows(st, seq, layers, heads, ln_eps=1e-5, log_prior=None, prior_row=None, alpha=0.0, log_prior2=None, prior_row2=None,
                       beta=0.0, first_col=0, dtype=torch.float32):
    """CPU statement of what ``pg_ar_loglik_fused`` must return for one unpadded sequence, following the semantics written in
    include/pgscore.h (pg_ar_fusion): log-softmax rows [len + 1, V] with, per predicted position t and vocabulary column
    v >= first_col, prior_row[t] >= 0 -> (1-alpha)*lp + alpha*log_prior[prior_row[t], v], then if prior_row2[t] >= 0
    -> (1-beta)*that + beta*log_prior2[prior_row2[t], v]; prior_row[t] == -2 -> (1-alpha)*lp. Returns (rows, sum of label terms).
    The mixing formulas are TranceptEVE's (trancepteve/model_pytorch.py:1113-1116, :1129-1133) in float32."""
    ids = torch.tensor([tokenize(seq)], dtype=torch.int64)
    with torch.no_grad():
        lp = torch.log_softmax(forward(st, ids, layers, heads, ln_eps, dtype)[0, :-1], dim=-1).float()
    fused = lp.clone()
    if prior_row is not None:
        P1 = torch.as_tensor(log_prior, dtype=torch.float32)
        P2 = torch.as_tensor(log_prior2, dtype=torch.float32) if log_prior2 is not None else None
        for t in range(lp.shape[0]):
            pr = int(prior_row[t])
            if pr >= 0:
                m = (1 - alpha) * lp[t, first_col:] + alpha * P1[pr, first_col:]
                if P2 is not None and int(prior_row2[t]) >= 0:
                    m = (1 - beta) * m + beta * P2[int(prior_row2[t]), first_col:]
                fused[t, first_col:] = m
            elif pr == -2:
                fused[t, first_col:] = (1 - alpha) * lp[t, first_col:]
    labels = ids[0, 1:]
    return fused.numpy(), float(fused.gather(1, labels[:, None]).sum())


def get_mutated_sequence(focus_seq, mutant, start_idx=1):
    """scoring_utils.py:16-31."""
    s = list(focus_seq)
    for m in mutant.split(":"):
        f, pos, t = m[0], int(m[1:-1]), m[-1]
        rel = pos - start_idx
        assert f == focus_seq[rel], "Invalid from_AA or mutant position: " + str(m) + " from_AA: " + str(f) + " relative pos: " + str(rel) + " focus_seq: " + str(focus_seq)
        assert t in AA_vocab, "Mutant to_AA is invalid: " + str(m)
        s[rel] = t
    return "".join(s)


def optimal_window(pos, L, W):
    """scoring_utils.py:47-60."""
    half = W // 2
    if L <= W:
        return [0, L]
    if pos < half:
        return [0, W]
    if pos >= L - half:
        return [L - W, L]
    return [max(0, pos - half), min(L, pos + half)]


def sequence_slices(df, target_seq, ctx, start_idx=1, scoring_window="optimal", indel_mode=False):
    """get_sequence_slices (scoring_utils.py:152-203) restated: rows (mutated_sequence, sliced_mutated_sequence, window_start,
    window_end) for mutants and matching WT windows, de-duplicated, original order."""
    L = len(target_seq)
    rows = []
    if scoring_window == "optimal":
        for mut, mseq in zip(df["mutant"], df["mutated_sequence"]):
            if indel_mode:
                ws, we = 0, len(mseq)
            else:
                bary = int(np.array([int(m[1:-1]) - start_idx for m in mut.split(":")]).mean())
                ws, we = optimal_window(bary, L, ctx)
            rows.append((mseq, mseq[ws:we], ws, we))
        wt = []
        for (_, _, ws, we) in rows:
            e = len(target_seq) if indel_mode else we
            wt.append((target_seq, target_seq[ws:e], ws, e))
        rows += wt
    else:
        nwin = 1 + int(L / ctx)
        start = 0
        for _ in range(nwin):
            blk = [(m, m[start:start + ctx], start, min(len(m), start + ctx)) for m in df["mutated_sequence"]]
            blk += [(target_seq, target_seq[start:start + ctx], start, min(len(target_seq), start + ctx)) for _ in df["mutated_sequence"]]
            rows += blk
            start += ctx
    out = pd.DataFrame(rows, columns=["mutated_sequence", "sliced_mutated_sequence", "window_start", "window_end"])
    return out.drop_duplicates().reset_index(drop=True)


def directional_scores(st, slices, target_seq, layers, heads, name, scoring_window="optimal", reverse=False, dtype=torch.float32,
                       ln_eps=1e-5, log_prior=None, alpha=0.6, msa_start=0, msa_end=None, rnd=None):
    """get_tranception_scores_mutated_sequences (scoring_utils.py:77-150): per-slice summed log-prob / len(full sequence),
    minus the WT scored in the same window (optimal) or the single WT reference (sliding)."""
    sc = slices.copy()
    cache = {}
    vals = []
    for s, ws, we in zip(sc["sliced_mutated_sequence"], sc["window_start"], sc["window_end"]):
        key = (s, ws, we)
        if key not in cache:
            with torch.no_grad():
                cache[key] = sequence_logprob(st, s[::-1] if reverse else s, layers, heads, ln_eps, dtype, log_prior, alpha, ws, we,
                                              msa_start, msa_end, reverse, rnd)
        vals.append(cache[key])
    sc["score"] = vals
    if scoring_window == "sliding":
        sc = sc[["mutated_sequence", "score"]].groupby("mutated_sequence").sum().reset_index()
    sc["score"] = sc["score"] / sc["mutated_sequence"].map(len)
    mut = sc[sc.mutated_sequence != target_seq]
    wt = sc[sc.mutated_sequence == target_seq]
    if scoring_window == "optimal":
        d = pd.merge(mut, wt, how="left", on=["window_start"], suffixes=("", "_wt"))
        d[name] = d["score"] - d["score_wt"]
    else:
        d = mut.copy()
        d[name] = d["score"] - list(wt["score"])[0]
    return d[["mutated_sequence", name]]


def score_mutants(st, DMS_data, target_seq, layers, heads, n_ctx=1024, scoring_mirror=True, indel_mode=False, scoring_window="optimal",
                  dtype=torch.float32, ln_eps=1e-5, log_prior=None, alpha=0.6, msa_start=0, msa_end=None, rnd=None):
    """TranceptionLMHeadModel.score_mutants (model_pytorch.py:878-928)."""
    df = DMS_data.copy()
    if "mutated_sequence" not in df and not indel_mode:
        df["mutated_sequence"] = df["mutant"].apply(lambda x: get_mutated_sequence(target_seq, x))
    assert "mutated_sequence" in df, "DMS file to score does not have mutated_sequence column"
    if "mutant" not in df:
        df["mutant"] = df["mutated_sequence"]
    df = df[["mutated_sequence", "mutant"]]
    sl = sequence_slices(df, target_seq, n_ctx - 2, scoring_window=scoring_window, indel_mode=indel_mode)
    kw = dict(scoring_window=scoring_window, dtype=dtype, ln_eps=ln_eps, log_prior=log_prior, alpha=alpha, msa_start=msa_start,
              msa_end=msa_end, rnd=rnd)
    out = directional_scores(st, sl, target_seq, layers, heads, "avg_score_L_to_R", **kw)
    if scoring_mirror:
        r = directional_scores(st, sl, target_seq, layers, heads, "avg_score_R_to_L", reverse=True, **kw)
        out = pd.merge(out, r, on="mutated_sequence", how="left", suffixes=("", "_R_to_L"))
        out["avg_score"] = (out["avg_score_L_to_R"] + out["avg_score_R_to_L"]) / 2.0
    else:
        out["avg_score"] = out["avg_score_L_to_R"]
    col = "mutant" if indel_mode else "mutated_sequence"
    if target_seq in DMS_data[col].values:
        row = pd.DataFrame([[target_seq, 0, 0, 0]] if scoring_mirror else [[target_seq, 0, 0]],
                           columns=[col, "avg_score_L_to_R", "avg_score_R_to_L", "avg_score"] if scoring_mirror else [col, "avg_score_L_to_R", "avg_score"])
        out = pd.concat([out, row], ignore_index=True)
    return out


# ----------------------------------------------------------------------------------------------------------------------
# MSA pre-processing (retrieval prior + sequence weights) — numpy restatements
def msa_prior(msa: dict, MSA_start, MSA_end, len_target_seq, weights=None, filter_MSA=True):
    """get_msa_prior, aggregate_substitution branch (tranception/utils/msa_utils.py:63-138). ``msa``: name -> aligned upper-case string."""
    vocab = {t: i for i, t in enumerate(VOCAB)}
    msa = dict(msa)
    def one_hot(s):
        o = np.zeros((len(s), len(vocab)))
        for j, c in enumerate(s):
            if c in vocab:
                o[j, vocab[c]] = 1.0
        return o.flatten()
    if filter_MSA:
        names = list(msa.keys())
        ref = one_hot(msa[names[0]])
        for n in names:
            if np.dot(ref, one_hot(msa[n])) / np.dot(ref, ref) < 0.2:
                del msa[n]
    if weights is not None:
        for n in list(msa.keys()):
            if n not in weights:
                del msa[n]
        w = [weights[n] for n in msa]
    else:
        w = [1] * len(msa)
    oh = np.zeros((len(msa), MSA_end - MSA_start, len(vocab)))
    for i, n in enumerate(msa):
        for j, c in enumerate(msa[n]):
            if c in vocab:
                oh[i, j, vocab[c]] = 1.0
    w = np.expand_dims(np.array(w), axis=(1, 2))
    weighted = (oh + 1e-5) * w
    norm = np.tile(weighted.sum(axis=-1).sum(axis=0).reshape(-1, 1), (1, len(vocab)))
    prior = np.zeros((len_target_seq, len(vocab)))
    prior[MSA_start:MSA_end, :] = weighted.sum(axis=0) / norm
    return prior


def cluster_weights(matrix, identity_threshold, empty_value=0):
    """calc_weights_fast + calc_num_cluster_members_nogaps (proteingym/utils/weights.py:13-53, :114-160)."""
    matrix = np.asarray(matrix)
    empty = np.all(matrix == empty_value, axis=1)
    act = matrix[~empty]
    N, L = act.shape
    Lng = 1.0 * L - np.sum(act == empty_value, axis=1)
    nn = np.ones(N)
    for i in range(N):
        eq = (act == act[i]) & (act[i] != empty_value)
        pm = eq.sum(axis=1)
        nn[i] += np.sum((pm / Lng[i] > identity_threshold) & (np.arange(N) != i))
    out = np.zeros(matrix.shape[0])
    out[~empty] = 1.0 / nn
    return out
