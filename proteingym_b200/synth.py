"""Seeded synthetic inputs at true architecture sizes.

There are no checkpoints, DMS CSVs or network in the build/GPU boxes (SURVEY.md §0.8), so parity and throughput
work uses:
  * synthetic fair-esm-format checkpoints (v1 = ESM-1b/ESM-1v ``{"args": Namespace, "model": state}``,
    v2 = ESM2 ``{"cfg": {"model": Namespace}, "model": state}``) that the *unmodified* reference loader accepts
    (reference: proteingym/baselines/esm/esm/pretrained.py:85-99,162-181,184-218), and
  * synthetic DMS tables / mapping files with the reference's column contract
    (reference: proteingym/baselines/esm/compute_fitness.py:288-326).

This module is product-side support code (used by bench.py, tests and the golden-vector scripts); it is NOT the
oracle and contains no scoring arithmetic.
"""
from __future__ import annotations

import argparse
import math
import os
from dataclasses import dataclass

import numpy as np
import torch

AA20 = "ACDEFGHIKLMNPQRSTVWY"


@dataclass
class EsmArch:
    kind: str  # "esm1v" (ESM-1b/ESM-1v: learned positions) | "esm2" (rotary)
    layers: int
    embed_dim: int
    heads: int
    ffn_dim: int
    token_dropout: bool = True
    emb_layer_norm_before: bool = False  # ESM-1b True, ESM-1v False (decided by key presence, pretrained.py:80-82)
    max_positions: int = 1024
    vocab: int = 33


ESM1V_650M = EsmArch("esm1v", 33, 1280, 20, 5120)
ESM1B_650M = EsmArch("esm1v", 33, 1280, 20, 5120, emb_layer_norm_before=True)
ESM2_8M = EsmArch("esm2", 6, 320, 20, 1280)      # head_dim 16
ESM2_35M = EsmArch("esm2", 12, 480, 20, 1920)    # head_dim 24, width not a multiple of 64
ESM2_150M = EsmArch("esm2", 30, 640, 20, 2560)   # head_dim 32
ESM2_650M = EsmArch("esm2", 33, 1280, 20, 5120)
ESM2_3B = EsmArch("esm2", 36, 2560, 40, 10240)


def _uniform(g, shape, bound):
    return (torch.rand(shape, generator=g, dtype=torch.float32, device=g.device) * 2 - 1) * bound


def make_esm_state(arch: EsmArch, seed: int = 0, qk_gain: float = 2.0, device=None) -> dict:
    """State dict with the key names of the reference modules (un-prefixed).

    Distributions follow the reference constructors' defaults (nn.Embedding N(0,1); nn.Linear U(+-1/sqrt(fan_in));
    q/k/v xavier-uniform with gain 1/sqrt(2), multihead_attention.py:138-155) except that biases and LayerNorm affine
    terms are made non-trivial so a dropped bias shows up in parity tests, and q/k are scaled by ``qk_gain`` so the
    attention softmax is far from uniform.

    ``device`` (default CPU) is where the tensors are drawn. The CPU stream is the one every golden fixture was generated from;
    a CUDA device gives the same distributions from a different stream in a fraction of the time (bench workloads at 3B size).
    """
    g = torch.Generator(device=device if device is not None else "cpu").manual_seed(seed)
    d, f, V = arch.embed_dim, arch.ffn_dim, arch.vocab
    st = {}
    # nn.Embedding's N(0,1) would give tied-output logits of std sqrt(d) (~36 at d=1280), far from a trained model's;
    # 0.1 keeps log-prob differences in the single digits like real ESM checkpoints.
    emb = 0.1 * torch.randn((V, d), generator=g, device=g.device)
    emb[1].zero_()  # padding_idx row (nn.Embedding(padding_idx=1))
    st["embed_tokens.weight"] = emb
    if arch.kind == "esm1v":
        pos = 0.1 * torch.randn((arch.max_positions + 2, d), generator=g, device=g.device)
        pos[1].zero_()
        st["embed_positions.weight"] = pos
        if arch.emb_layer_norm_before:
            st["emb_layer_norm_before.weight"] = 1 + 0.1 * torch.randn(d, generator=g, device=g.device)
            st["emb_layer_norm_before.bias"] = 0.05 * torch.randn(d, generator=g, device=g.device)
    for i in range(arch.layers):
        p = f"layers.{i}."
        xb = math.sqrt(3.0 / (2 * d))  # xavier_uniform gain 1/sqrt(2): sqrt(6/(2d))/sqrt(2)
        for nm, gain in (("q", qk_gain), ("k", qk_gain), ("v", 1.0)):
            st[p + f"self_attn.{nm}_proj.weight"] = _uniform(g, (d, d), xb) * gain
            st[p + f"self_attn.{nm}_proj.bias"] = _uniform(g, (d,), 1 / math.sqrt(d)) * gain
        st[p + "self_attn.out_proj.weight"] = _uniform(g, (d, d), math.sqrt(6.0 / (2 * d)))
        st[p + "self_attn.out_proj.bias"] = _uniform(g, (d,), 1 / math.sqrt(d))
        st[p + "self_attn_layer_norm.weight"] = 1 + 0.1 * torch.randn(d, generator=g, device=g.device)
        st[p + "self_attn_layer_norm.bias"] = 0.05 * torch.randn(d, generator=g, device=g.device)
        st[p + "fc1.weight"] = _uniform(g, (f, d), 1 / math.sqrt(d))
        st[p + "fc1.bias"] = _uniform(g, (f,), 1 / math.sqrt(d))
        st[p + "fc2.weight"] = _uniform(g, (d, f), 1 / math.sqrt(f))
        st[p + "fc2.bias"] = _uniform(g, (d,), 1 / math.sqrt(f))
        st[p + "final_layer_norm.weight"] = 1 + 0.1 * torch.randn(d, generator=g, device=g.device)
        st[p + "final_layer_norm.bias"] = 0.05 * torch.randn(d, generator=g, device=g.device)
        if arch.kind == "esm2":
            hd = d // arch.heads
            st[p + "self_attn.rot_emb.inv_freq"] = (1.0 / (10000 ** (torch.arange(0, hd, 2).float() / hd))).to(g.device)
    st["emb_layer_norm_after.weight"] = 1 + 0.1 * torch.randn(d, generator=g, device=g.device)
    st["emb_layer_norm_after.bias"] = 0.05 * torch.randn(d, generator=g, device=g.device)
    st["lm_head.dense.weight"] = _uniform(g, (d, d), 1 / math.sqrt(d))
    st["lm_head.dense.bias"] = _uniform(g, (d,), 1 / math.sqrt(d))
    st["lm_head.layer_norm.weight"] = 1 + 0.1 * torch.randn(d, generator=g, device=g.device)
    st["lm_head.layer_norm.bias"] = 0.05 * torch.randn(d, generator=g, device=g.device)
    st["lm_head.bias"] = 0.1 * torch.randn(V, generator=g, device=g.device)
    # tied: same tensor object, so torch.save keeps the aliasing like the released checkpoints do
    st["lm_head.weight"] = st["embed_tokens.weight"]
    return st


def write_esm_checkpoint(path: str, arch: EsmArch, seed: int = 0, state: dict | None = None) -> dict:
    """Write ``state`` (or a fresh seeded one) in the fair-esm on-disk format the reference loader dispatches on:
    file stem starting with ``esm2`` -> v2, anything else -> v1 (pretrained.py:184-188)."""
    st = state if state is not None else make_esm_state(arch, seed)
    stem = os.path.basename(path)
    if arch.kind == "esm2":
        assert stem.startswith("esm2"), "reference dispatches v2 on the file name (pretrained.py:187)"
        assert arch.ffn_dim == 4 * arch.embed_dim, "ESM2 hard-codes ffn = 4 * embed_dim (esm2.py:52)"
        cfg = argparse.Namespace(encoder_layers=arch.layers, encoder_embed_dim=arch.embed_dim,
                                 encoder_attention_heads=arch.heads, token_dropout=arch.token_dropout)
        blob = {"cfg": {"model": cfg},
                "model": {("encoder.lm_head." + k[len("lm_head."):] if k.startswith("lm_head.")
                           else "encoder.sentence_encoder." + k): v for k, v in st.items()}}
    else:
        assert not stem.startswith("esm2")
        args = argparse.Namespace(arch="roberta_large", layers=arch.layers, embed_dim=arch.embed_dim,
                                  ffn_embed_dim=arch.ffn_dim, attention_heads=arch.heads,
                                  max_positions=arch.max_positions, token_dropout=arch.token_dropout,
                                  final_bias=True)
        blob = {"args": args,
                "model": {("encoder.lm_head." + k[len("lm_head."):] if k.startswith("lm_head.")
                           else "encoder.sentence_encoder." + k): v for k, v in st.items()}}
    torch.save(blob, path)
    return st


def random_protein(L: int, seed: int) -> str:
    rng = np.random.RandomState(seed)
    return "".join(AA20[i] for i in rng.randint(0, 20, size=L))


def all_single_mutants(seq: str, first: int = 1, last: int | None = None, offset: int = 1):
    """All 19 substitutions at (1-based, offset-adjusted) positions first..last."""
    last = len(seq) if last is None else last
    out = []
    for pos in range(first, last + 1):
        wt = seq[pos - offset]
        for a in AA20:
            if a != wt:
                out.append(f"{wt}{pos}{a}")
    return out


def sample_mutants(seq: str, n: int, seed: int, multi_frac: float = 0.0, max_sites: int = 5, offset: int = 1):
    """Uniform sample without replacement from the 19*L singles (SURVEY.md §8d config 2); a fraction
    ``multi_frac`` of rows are turned into 2..max_sites multi-mutants ("A24G:T30S")."""
    rng = np.random.RandomState(seed)
    singles = all_single_mutants(seq, offset=offset)
    idx = rng.choice(len(singles), size=min(n, len(singles)), replace=False)
    muts = [singles[i] for i in idx]
    if multi_frac > 0:
        for r in range(len(muts)):
            if rng.rand() < multi_frac:
                k = rng.randint(2, max_sites + 1)
                pos = rng.choice(len(seq), size=k, replace=False)
                parts = []
                for p in sorted(pos):
                    wt = seq[p]
                    mt = AA20[rng.randint(0, 20)]
                    while mt == wt:
                        mt = AA20[rng.randint(0, 20)]
                    parts.append(f"{wt}{p + offset}{mt}")
                muts[r] = ":".join(parts)
    return muts


def apply_mutant(seq: str, mutant: str, offset: int = 1) -> str:
    s = list(seq)
    for m in mutant.split(":"):
        wt, pos, mt = m[0], int(m[1:-1]) - offset, m[-1]
        assert s[pos] == wt
        s[pos] = mt
    return "".join(s)


def write_dms_csv(path: str, seq: str, mutants, seed: int = 0):
    """DMS CSV with the reference's columns (mutant, mutated_sequence, DMS_score, DMS_score_bin)."""
    import pandas as pd
    rng = np.random.RandomState(seed)
    score = rng.randn(len(mutants))
    df = pd.DataFrame({"mutant": mutants,
                       "mutated_sequence": [apply_mutant(seq, m) for m in mutants],
                       "DMS_score": score,
                       "DMS_score_bin": (score > 0).astype(int)})
    df.to_csv(path, index=False)
    return df


def write_mapping_csv(path: str, rows):
    """Reference-file CSV with the columns compute_fitness.main reads (compute_fitness.py:288-307):
    rows = [(DMS_id, DMS_filename, target_seq), ...]."""
    import pandas as pd
    df = pd.DataFrame({"DMS_id": [r[0] for r in rows], "DMS_filename": [r[1] for r in rows],
                       "target_seq": [r[2] for r in rows]})
    df.to_csv(path, index=False)
    return df


# ----------------------------------------------------------------------------------------------------------------------
# Tranception (reference: proteingym/baselines/tranception/tranception/model_pytorch.py, config.py)
@dataclass
class TranceptionArch:
    layers: int
    embed_dim: int
    heads: int          # multiple of 4 (grouped ALiBi / depthwise-conv head groups, model_pytorch.py:129-131)
    ffn_dim: int        # n_inner (None in config.json means 4 * n_embd, model_pytorch.py:284)
    n_ctx: int = 1024
    vocab: int = 25
    ln_eps: float = 1e-5


TRANCEPTION_L = TranceptionArch(36, 1280, 20, 5120)


def make_tranception_state(arch: TranceptionArch, seed: int = 0, qk_gain: float = 3.0) -> dict:
    """HF-style state dict keys of ``TranceptionLMHeadModel`` (GPT2 naming; Conv1D weights are [in, out])."""
    g = torch.Generator().manual_seed(seed)
    d, f, V, hd = arch.embed_dim, arch.ffn_dim, arch.vocab, arch.embed_dim // arch.heads
    st = {"transformer.wte.weight": 0.1 * torch.randn((V, d), generator=g)}
    for i in range(arch.layers):
        p = f"transformer.h.{i}."
        st[p + "ln_1.weight"] = 1 + 0.1 * torch.randn(d, generator=g)
        st[p + "ln_1.bias"] = 0.05 * torch.randn(d, generator=g)
        w = torch.randn((d, 3 * d), generator=g) / math.sqrt(d)
        w[:, :2 * d] *= qk_gain / 2
        st[p + "attn.c_attn.weight"] = w
        st[p + "attn.c_attn.bias"] = 0.1 * torch.randn(3 * d, generator=g)
        st[p + "attn.c_proj.weight"] = torch.randn((d, d), generator=g) / math.sqrt(d)
        st[p + "attn.c_proj.bias"] = 0.05 * torch.randn(d, generator=g)
        for nm in ("query", "key", "value"):
            for ki, k in enumerate((3, 5, 7)):
                st[p + f"attn.{nm}_depthwiseconv.{ki}.conv.weight"] = torch.randn((hd, 1, k), generator=g) / math.sqrt(k)
                st[p + f"attn.{nm}_depthwiseconv.{ki}.conv.bias"] = 0.1 * torch.randn(hd, generator=g)
        st[p + "ln_2.weight"] = 1 + 0.1 * torch.randn(d, generator=g)
        st[p + "ln_2.bias"] = 0.05 * torch.randn(d, generator=g)
        st[p + "mlp.c_fc.weight"] = torch.randn((d, f), generator=g) / math.sqrt(d)
        st[p + "mlp.c_fc.bias"] = 0.1 * torch.randn(f, generator=g)
        st[p + "mlp.c_proj.weight"] = torch.randn((f, d), generator=g) / math.sqrt(f) * 0.5
        st[p + "mlp.c_proj.bias"] = 0.05 * torch.randn(d, generator=g)
    st["transformer.ln_f.weight"] = 1 + 0.1 * torch.randn(d, generator=g)
    st["transformer.ln_f.bias"] = 0.05 * torch.randn(d, generator=g)
    st["lm_head.weight"] = st["transformer.wte.weight"]  # tied (GPT2 ties input and output embeddings)
    return st


def write_tranception_checkpoint(folder: str, arch: TranceptionArch, seed: int = 0, state: dict | None = None) -> dict:
    """HF checkpoint directory: config.json + pytorch_model.bin (what score_tranception_proteingym.py:79,100 reads)."""
    import json
    os.makedirs(folder, exist_ok=True)
    st = state if state is not None else make_tranception_state(arch, seed)
    cfg = {"n_embd": arch.embed_dim, "n_head": arch.heads, "n_layer": arch.layers, "n_ctx": arch.n_ctx, "n_positions": arch.n_ctx,
           "n_inner": arch.ffn_dim, "vocab_size": arch.vocab, "layer_norm_epsilon": arch.ln_eps, "activation_function": "squared_relu",
           "attention_mode": "tranception", "position_embedding": "grouped_alibi", "scale_attn_weights": True,
           "architectures": ["TranceptionLMHeadModel"], "model_type": "tranception"}
    with open(os.path.join(folder, "config.json"), "w") as fh:
        json.dump(cfg, fh, indent=1)
    torch.save(st, os.path.join(folder, "pytorch_model.bin"))
    return st


def random_indels(seq: str, n: int, seed: int, max_len: int = 4):
    """Synthetic indel variants of ``seq`` (full mutated sequences, as the DMS_indels files list them)."""
    rng = np.random.RandomState(seed)
    out = set()
    while len(out) < n:
        pos = rng.randint(0, len(seq))
        k = rng.randint(1, max_len + 1)
        if rng.rand() < 0.5:
            s = seq[:pos] + "".join(AA20[i] for i in rng.randint(0, 20, size=k)) + seq[pos:]
        else:
            s = seq[:pos] + seq[pos + k:]
        if s != seq and len(s) > 2:
            out.add(s)
    return sorted(out)


def synthetic_msa(target_seq: str, n: int, seed: int, sub_rate=(0.05, 0.9), gap_rate=0.1, gappy_cols=(), gappy_rate=0.6):
    """name -> aligned sequence (a2m-like, upper case, '-' gaps, occasional 'X'); first entry is the target itself.
    ``gappy_cols`` get gaps at ``gappy_rate`` instead (columns that fall below a focus-column occupancy threshold)."""
    rng = np.random.RandomState(seed)
    msa = {">target/1-%d" % len(target_seq): target_seq}
    gappy = set(gappy_cols)
    for i in range(n - 1):
        r = rng.uniform(*sub_rate)
        s = list(target_seq)
        for j in range(len(s)):
            u = rng.rand()
            if u < (gappy_rate if j in gappy else gap_rate):
                s[j] = "-"
            elif u < gap_rate + r:
                s[j] = AA20[rng.randint(0, 20)] if rng.rand() > 0.02 else "X"
        msa[">seq%d" % i] = "".join(s)
    return msa


# EVE VAE (trancepteve/EVE/VAE_model.py) at toy width: same keys as utils/eve_model_default_params.json
EVE_TINY_PARAMS = {
    "encoder_parameters": {"hidden_layers_sizes": [48, 32, 24], "z_dim": 8, "convolve_input": False, "convolution_input_depth": 40,
                           "nonlinear_activation": "relu", "dropout_proba": 0.0},
    "decoder_parameters": {"hidden_layers_sizes": [24, 32, 50], "z_dim": 8, "bayesian_decoder": True, "first_hidden_nonlinearity": "relu",
                           "last_hidden_nonlinearity": "relu", "dropout_proba": 0.1, "convolve_output": True, "convolution_output_depth": 10,
                           "include_temperature_scaler": True, "include_sparsity": False, "num_tiles_sparsity": 0, "logit_sparsity_p": 0},
}


def make_eve_state(seq_len: int, params: dict = None, seed: int = 0, log_var: float = -4.0) -> dict:
    """Seeded ``model_state_dict`` of the reference's EVE ``VAE_model`` (MLP encoder + Bayesian MLP decoder with 1x1 output
    convolution and temperature scaler; key names/shapes as VAE_encoder.py:40-52, VAE_decoder.py:47-108). ``log_var`` sets every
    weight-posterior log-variance (the reference initialises them to -10; a larger value makes the sampling noise visible)."""
    params = params or EVE_TINY_PARAMS
    g = torch.Generator().manual_seed(seed)
    A = 20
    enc, dec = params["encoder_parameters"], params["decoder_parameters"]

    def lin(o, i):
        return torch.randn((o, i), generator=g) / math.sqrt(i), 0.1 + 0.05 * torch.randn(o, generator=g)

    st = {}
    sizes = [A * seq_len] + list(enc["hidden_layers_sizes"])
    for k in range(len(sizes) - 1):
        st[f"encoder.hidden_layers.{k}.weight"], st[f"encoder.hidden_layers.{k}.bias"] = lin(sizes[k + 1], sizes[k])
    st["encoder.fc_mean.weight"], st["encoder.fc_mean.bias"] = lin(enc["z_dim"], sizes[-1])
    w, _ = lin(enc["z_dim"], sizes[-1])
    st["encoder.fc_log_var.weight"], st["encoder.fc_log_var.bias"] = 0.1 * w, torch.full((enc["z_dim"],), -2.0)
    H = dec["hidden_layers_sizes"]
    C = dec["convolution_output_depth"] if dec["convolve_output"] else A
    st["decoder.last_hidden_layer_weight_mean"] = torch.randn((C * seq_len, H[-1]), generator=g) * math.sqrt(2.0 / (C * seq_len + H[-1]))
    st["decoder.last_hidden_layer_weight_log_var"] = torch.full((C * seq_len, H[-1]), log_var)
    st["decoder.last_hidden_layer_bias_mean"] = 0.1 + 0.3 * torch.randn(A * seq_len, generator=g)
    st["decoder.last_hidden_layer_bias_log_var"] = torch.full((A * seq_len,), log_var)
    if dec["include_temperature_scaler"]:
        st["decoder.temperature_scaler_mean"] = torch.ones(1) * 2.0
        st["decoder.temperature_scaler_log_var"] = torch.full((1,), log_var)
    dsz = [dec["z_dim"]] + list(H)
    for k in range(len(H)):
        st[f"decoder.hidden_layers_mean.{k}.weight"], st[f"decoder.hidden_layers_mean.{k}.bias"] = lin(dsz[k + 1], dsz[k])
        st[f"decoder.hidden_layers_log_var.{k}.weight"] = torch.full((dsz[k + 1], dsz[k]), log_var)
        st[f"decoder.hidden_layers_log_var.{k}.bias"] = torch.full((dsz[k + 1],), log_var)
    if dec["convolve_output"]:
        st["decoder.output_convolution_mean.weight"] = torch.randn((A, C, 1), generator=g) / math.sqrt(C) * 3.0
        st["decoder.output_convolution_log_var.weight"] = torch.full((A, C, 1), log_var)
    return st


def write_a2m(path: str, msa: dict, width: int = 60):
    with open(path, "w") as fh:
        for n, s in msa.items():
            fh.write(n + "\n")
            for k in range(0, len(s), width):
                fh.write(s[k:k + width] + "\n")


# ----------------------------------------------------------------------------------------------------------------------
# MSA Transformer (reference: proteingym/baselines/esm/esm/model/msa_transformer.py, esm/axial_attention.py, esm/modules.py:145-235)
@dataclass
class MsaArch:
    layers: int
    embed_dim: int
    heads: int
    ffn_dim: int
    embed_positions_msa: bool = True
    msa_pos_dim: int = 0       # last dimension of msa_position_embedding: 0 = embed_dim (MSA-1b), 1 = the first release's broadcast form
    max_positions: int = 1024
    vocab: int = 33


MSA_1B = MsaArch(12, 768, 12, 3072)


def make_msa_state(arch: MsaArch, seed: int = 0, qk_gain: float = 2.0, device=None) -> dict:
    """State dict with the key names of the reference ``MSATransformer`` module (msa_transformer.py:100-148; AxialTransformerLayer
    = three NormalizedResidualBlocks, modules.py:194-203,374-388). Same distributions as ``make_esm_state``."""
    g = torch.Generator(device=device if device is not None else "cpu").manual_seed(seed)
    d, f, V = arch.embed_dim, arch.ffn_dim, arch.vocab
    rn = lambda *shape: torch.randn(shape, generator=g, device=g.device)
    st = {}
    emb = 0.1 * rn(V, d)
    emb[1].zero_()
    st["embed_tokens.weight"] = emb
    if arch.embed_positions_msa:
        st["msa_position_embedding"] = 0.1 * rn(1, 1024, 1, arch.msa_pos_dim or d)
    pos = 0.1 * rn(arch.max_positions + 2, d)
    pos[1].zero_()
    st["embed_positions.weight"] = pos
    st["emb_layer_norm_before.weight"] = 1 + 0.1 * rn(d)
    st["emb_layer_norm_before.bias"] = 0.05 * rn(d)
    xb = math.sqrt(3.0 / (2 * d))
    for i in range(arch.layers):
        for blk in ("row_self_attention", "column_self_attention"):
            p = f"layers.{i}.{blk}."
            for nm, gain in (("k", qk_gain), ("v", 1.0), ("q", qk_gain)):
                st[p + f"layer.{nm}_proj.weight"] = _uniform(g, (d, d), xb) * gain
                st[p + f"layer.{nm}_proj.bias"] = _uniform(g, (d,), 1 / math.sqrt(d)) * gain
            st[p + "layer.out_proj.weight"] = _uniform(g, (d, d), math.sqrt(6.0 / (2 * d)))
            st[p + "layer.out_proj.bias"] = _uniform(g, (d,), 1 / math.sqrt(d))
            st[p + "layer_norm.weight"] = 1 + 0.1 * rn(d)
            st[p + "layer_norm.bias"] = 0.05 * rn(d)
        p = f"layers.{i}.feed_forward_layer."
        st[p + "layer.fc1.weight"] = _uniform(g, (f, d), 1 / math.sqrt(d))
        st[p + "layer.fc1.bias"] = _uniform(g, (f,), 1 / math.sqrt(d))
        st[p + "layer.fc2.weight"] = _uniform(g, (d, f), 1 / math.sqrt(f))
        st[p + "layer.fc2.bias"] = _uniform(g, (d,), 1 / math.sqrt(f))
        st[p + "layer_norm.weight"] = 1 + 0.1 * rn(d)
        st[p + "layer_norm.bias"] = 0.05 * rn(d)
    st["emb_layer_norm_after.weight"] = 1 + 0.1 * rn(d)
    st["emb_layer_norm_after.bias"] = 0.05 * rn(d)
    st["lm_head.dense.weight"] = _uniform(g, (d, d), 1 / math.sqrt(d))
    st["lm_head.dense.bias"] = _uniform(g, (d,), 1 / math.sqrt(d))
    st["lm_head.layer_norm.weight"] = 1 + 0.1 * rn(d)
    st["lm_head.layer_norm.bias"] = 0.05 * rn(d)
    st["lm_head.bias"] = 0.1 * rn(V)
    st["lm_head.weight"] = st["embed_tokens.weight"]
    return st


def msa_file_key(model_key: str) -> str:
    """Model key -> key in a released msa_transformer checkpoint file: the loader swaps "row" and "column" in every name
    (pretrained.py:113,115) and strips the ``encoder.`` / ``encoder.sentence_encoder.`` prefixes (:109-112)."""
    k = model_key.replace("row", "\0").replace("column", "row").replace("\0", "column")
    return ("encoder.lm_head." + k[len("lm_head."):]) if k.startswith("lm_head.") else "encoder.sentence_encoder." + k


def write_msa_checkpoint(path: str, arch: MsaArch, seed: int = 0, state: dict | None = None) -> dict:
    """fair-esm v1 file (``{"args": Namespace(arch="msa_transformer", ...), "model": state}``) that the reference loader accepts."""
    st = state if state is not None else make_msa_state(arch, seed)
    assert not os.path.basename(path).startswith("esm2")
    args = argparse.Namespace(arch="msa_transformer", layers=arch.layers, embed_dim=arch.embed_dim, ffn_embed_dim=arch.ffn_dim,
                              attention_heads=arch.heads, max_positions=arch.max_positions, dropout=0.1, attention_dropout=0.1,
                              activation_dropout=0.1, max_tokens=2 ** 14, max_tokens_per_msa=2 ** 14, embed_positions_msa=arch.embed_positions_msa,
                              final_bias=True)
    torch.save({"args": args, "model": {msa_file_key(k): v for k, v in st.items()}}, path)
    return st


def random_alignment(target_seq: str, n_rows: int, seed: int, sub_rate=(0.05, 0.6), gap_rate: float = 0.08, insert_cols=()):
    """[(name, aligned row)] for the MSA Transformer path: the target first (name ``>target/1-L``), rows of the same length made of
    upper-case residues and '-' (and '.' in ``insert_cols`` of the non-target rows, which the reference keeps as tokens after
    upper-casing, compute_fitness.py:69-70)."""
    rng = np.random.RandomState(seed)
    rows = [(">target/1-%d" % len(target_seq), target_seq)]
    ins = set(insert_cols)
    for i in range(n_rows - 1):
        r = rng.uniform(*sub_rate)
        s = list(target_seq)
        for j in range(len(s)):
            u = rng.rand()
            if j in ins:
                s[j] = "."
            elif u < gap_rate:
                s[j] = "-"
            elif u < gap_rate + r:
                s[j] = AA20[rng.randint(0, 20)]
        rows.append((">seq%d/1-%d" % (i, len(target_seq)), "".join(s)))
    return rows
