"""CPU: the small ESM2 releases (8M, 35M, 150M).
  * oracle/esm_oracle.py reproduces the goldens the unmodified reference produced at their true shapes;
  * the operand layout the library packs for them (api.cu OpFmt and slot maps: 64-wide head slots, q/k rotate-half halves at slot
    columns 0 and 32, GEMM inputs zero-padded to a multiple of 64, [T, 32] rotary tables) gives, in fp64, the attention block of the
    reference MultiheadAttention with rotary embeddings (multihead_attention.py:242-395) for head dims 16, 24 and 32."""
import math

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import esm_oracle as O
from oracle import ref_shims


@pytest.mark.parametrize("name", ["esm2_8m", "esm2_35m", "esm2_150m", "esm2_8m_window"])
def test_oracle_matches_reference_goldens(name):
    g = load_golden(name)
    arch, seq, meta = g["arch"], g["seq"], g["meta"]
    pos = meta.get("table_positions") or [1, len(seq) // 2, len(seq)]
    table = O.masked_marginal_table(O.load_state(g["state"](), "esm2"), seq, "esm2", arch.layers, arch.heads, positions=pos, batch=16)
    want = g["table"] if "table_positions" in meta else g["table"][pos]
    assert np.abs(table[pos].numpy() - want).max() < 5e-5
    if name == "esm2_8m":  # every row, and the reference CLI's scores
        table = O.masked_marginal_table(O.load_state(g["state"](), "esm2"), seq, "esm2", arch.layers, arch.heads, batch=16)
        assert np.abs(table.numpy() - g["table"]).max() < 5e-5
        col = meta["ckpt_names"][0].split(".")[0]
        assert np.abs(O.score_mutants(g["df"]["mutant"], seq, table) - g["df"][col].to_numpy()).max() < 1e-4


def slot_src(i, kind, n, hd):
    """api.cu slot_src: index i of a padded width -> source index, or -1 for a zero."""
    if kind == "pad":
        return i if i < n else -1
    h, c = divmod(i, 64)
    if kind == "head":
        return h * hd + c if c < hd else -1
    half = hd // 2
    return h * hd + c if c < half else (h * hd + half + c - 32 if 32 <= c < 32 + half else -1)


def expand(w, N, K, rkind, ckind, hd):
    """api.cu expand_slots_kernel: [n, k] -> [N, K] with rows / columns placed by slot maps, zeros elsewhere."""
    w = torch.nn.functional.pad(w.reshape(w.shape[0], -1), (0, 1, 0, 1))  # index -1 reads the appended zero row / column
    rows = torch.tensor([slot_src(i, rkind, w.shape[0] - 1, hd) for i in range(N)])
    return w[rows][:, torch.tensor([slot_src(j, ckind, w.shape[1] - 1, hd) for j in range(K)])]


def slotted_attention(x, p, heads, hd, inv_freq):
    """The block as the library computes it: QKV on dk-padded inputs into head slots, the GEMM's rotary epilogue on slot pairs
    (c, c + 32) with [T, 32] tables zero after hd/2, 64-wide attention per slot, out_proj with K = heads * 64."""
    T, d = x.shape
    da, dk, s = heads * 64, (d + 63) // 64 * 64, 1.0 / math.sqrt(hd)
    xa = torch.cat([x, torch.zeros((T, dk - d), dtype=x.dtype)], 1)
    def proj(n, kind, sc=1.0):  # q: hd^-1/2 folded into weights and bias, as pg_load_weights does
        return xa @ (expand(p[n + ".weight"], da, dk, kind, "pad", hd) * sc).T + expand(p[n + ".bias"], da, 1, kind, "pad", hd)[:, 0] * sc
    q, k, v = proj("q_proj", "rot", s), proj("k_proj", "rot"), proj("v_proj", "head").view(T, heads, 64)
    freqs = torch.arange(T, dtype=inv_freq.dtype)[:, None] * inv_freq[None, :]  # checkpoint.rotary_tables: [T, hd/2]
    cos, sin = torch.zeros((T, 1, 32), dtype=x.dtype), torch.zeros((T, 1, 32), dtype=x.dtype)
    cos[:, 0, :hd // 2], sin[:, 0, :hd // 2] = freqs.cos(), freqs.sin()
    rot = lambda y: (lambda a, b: torch.cat([a * cos - b * sin, b * cos + a * sin], -1))(*y.view(T, heads, 64).split(32, -1))
    o = torch.einsum("hts,shc->thc", torch.softmax(torch.einsum("thc,shc->hts", rot(q), rot(k)), -1), v)
    assert torch.all(o[..., hd:] == 0)  # the padding columns of every slot stay exact zeros
    return o.reshape(T, da) @ expand(p["out_proj.weight"], d, da, "pad", "head", hd).T + p["out_proj.bias"]


@pytest.mark.parametrize("hd,heads", [(16, 20), (24, 20), (32, 20), (64, 2)])
def test_slot_layout_matches_attention_block_fp64(hd, heads):
    """(24, 20) is ESM2 35M: d = 480, so the inputs are padded to 512 columns too. (64, 2): the unpadded layout."""
    d = hd * heads
    g = torch.Generator().manual_seed(hd)
    p = {f"{n}_proj.{t}": torch.randn((d, d) if t == "weight" else (d,), generator=g, dtype=torch.float64) / math.sqrt(d)
         for n in ("q", "k", "v", "out") for t in ("weight", "bias")}
    x = torch.randn((37, d), generator=g, dtype=torch.float64)
    inv_freq = 1.0 / (10000 ** (torch.arange(0, hd, 2).float() / hd))  # rotary_embedding.py:37-38, fp32 as in checkpoints
    # esm_oracle's restatement (q scaled after the projection, rotate_half over hd-wide heads)
    q, k, v = ((x @ p[f"{n}_proj.weight"].T + p[f"{n}_proj.bias"]).view(37, heads, hd).transpose(0, 1) for n in "qkv")
    freqs = torch.arange(37).float()[:, None] * inv_freq[None, :]
    cos, sin = torch.cat([freqs, freqs], -1).cos().double(), torch.cat([freqs, freqs], -1).sin().double()
    q, k = (q * hd ** -0.5) * cos + O.rotate_half(q * hd ** -0.5) * sin, k * cos + O.rotate_half(k) * sin
    want = (torch.softmax(q @ k.transpose(-1, -2), -1) @ v).transpose(0, 1).reshape(37, d) @ p["out_proj.weight"].T + p["out_proj.bias"]
    assert (slotted_attention(x, p, heads, hd, inv_freq) - want).abs().max().item() < 1e-12
    if ref_shims.available():  # the reference module itself, where the reference tree is present
        ref_shims.install()
        from esm.multihead_attention import MultiheadAttention
        m = MultiheadAttention(d, heads, use_rotary_embeddings=True).double().eval()
        with torch.no_grad():
            for n in ("q", "k", "v", "out"):
                getattr(m, f"{n}_proj").weight.copy_(p[f"{n}_proj.weight"])
                getattr(m, f"{n}_proj").bias.copy_(p[f"{n}_proj.bias"])
            m.rot_emb.inv_freq.copy_(inv_freq.double())
            ref, _ = m(x[:, None], x[:, None], x[:, None], need_weights=False)
        # the module builds fp64 tables (so do we here) but runs its softmax in fp32 (utils_softmax): hence 1e-6
        assert (slotted_attention(x, p, heads, hd, inv_freq.double()) - ref[:, 0]).abs().max().item() < 1e-6
