"""ORACLE — a plain-torch restatement of PoET's scoring forward (poet/models/poet.py PoET.embed / logits,
modules/transformer.py TieredTransformerEncoderLayer, modules/embedding.py RotaryEmbedding) in any dtype (fp64 for the GPU tests), on any
device. Written from the reference's equations, not copied: token embedding without positions; per layer a causal self-attention within
each sequence, a causal attention over the whole sequence of sequences, and an erf-GELU MLP, each pre-LN and residual; interleaved rotary
over 64-wide heads with positions restarting at 0 in every sequence; softmax scale 1/sqrt(64); then `norm` (LayerNorm or identity) and the
24-way head. ``context`` returns the per-layer record (rotated multi-attention keys, values); ``token_logp`` scores variant rows against
it with the mask token (23) ignored as CrossEntropyLoss(ignore_index=23) does. Queries are chunked so that a 24 640-row context fits."""
from __future__ import annotations

import torch
import torch.nn.functional as F

MASK = 23
Q_CHUNK = 1024


class PoetOracle:
    def __init__(self, state: dict, layers: int, heads: int, dtype=torch.float64, device="cpu"):
        self.w = {k: v.to(device, dtype) for k, v in state.items()}
        self.inv = state["rotary_emb.inv_freq"].to(device, torch.float64)
        self.L, self.H, self.dtype, self.device = layers, heads, dtype, device
        self.norm = "norm.weight" in state

    def _ln(self, x, p):
        return F.layer_norm(x, x.shape[-1:], self.w[p + ".weight"], self.w[p + ".bias"], 1e-5)

    def _rot(self, x, pos):  # x [n, H, 64]; pairs (2i, 2i+1) rotated by pos * inv_freq[2i]
        f = (pos.to(torch.float64)[:, None] * self.inv[None, :]).to(self.dtype)
        cos, sin = torch.cos(f)[:, None, :], torch.sin(f)[:, None, :]
        x2 = x.unflatten(-1, (-1, 2))
        rh = torch.stack((-x2[..., 1], x2[..., 0]), dim=-1).flatten(-2)
        return x * cos + rh * sin

    def _qkv(self, x, p, pos):
        n = x.shape[0]
        q = (x @ self.w[p + "q_proj.weight"].T).view(n, self.H, -1)
        k = (x @ self.w[p + "k_proj.weight"].T).view(n, self.H, -1)
        v = (x @ self.w[p + "v_proj.weight"].T).view(n, self.H, -1)
        return self._rot(q, pos), self._rot(k, pos), v

    def _attn(self, q, k, v, visible):  # visible(rows) -> bool [len(rows), nk]
        out = torch.empty_like(q)
        kt, vt = k.transpose(0, 1), v.transpose(0, 1)
        for a in range(0, q.shape[0], Q_CHUNK):
            rows = torch.arange(a, min(a + Q_CHUNK, q.shape[0]), device=self.device)
            s = torch.matmul(q[rows].transpose(0, 1), kt.transpose(1, 2)) * (q.shape[-1] ** -0.5)
            s = s.masked_fill(~visible(rows)[None], float("-inf"))
            out[rows] = torch.matmul(torch.softmax(s, dim=-1), vt).transpose(0, 1)
        return out

    def _out(self, o, p):
        return o.flatten(1) @ self.w[p + "out_proj.weight"].T + self.w[p + "out_proj.bias"]

    def _mlp(self, x, p):
        h = F.gelu(self._ln(x, p + "norm3") @ self.w[p + "linear1.weight"].T + self.w[p + "linear1.bias"])
        return h @ self.w[p + "linear2.weight"].T + self.w[p + "linear2.bias"]

    def context(self, ids: torch.Tensor, seg_lens: list[int]):
        """-> [(k, v)] per layer: the multi-sequence attention's rotated keys and values of the packed context, [Tm, H, 64] each."""
        pos = torch.cat([torch.arange(n) for n in seg_lens]).to(self.device)
        seg = torch.cat([torch.full((n,), s) for n, s in zip(seg_lens, [0] + list(torch.tensor(seg_lens).cumsum(0)[:-1].tolist()))])
        seg = seg.to(self.device)
        Tm = len(pos)
        keys = torch.arange(Tm, device=self.device)
        x = self.w["token_embed.weight"][ids.to(self.device)]
        rec = []
        for l in range(self.L):
            p = f"decoder.layers.{l}."
            q, k, v = self._qkv(self._ln(x, p + "norm1"), p + "self_attn.", pos)
            x = x + self._out(self._attn(q, k, v, lambda r: (keys[None] <= r[:, None]) & (keys[None] >= seg[r][:, None])), p + "self_attn.")
            q, k, v = self._qkv(self._ln(x, p + "norm2"), p + "multihead_attn.", pos)
            rec.append((k, v))
            x = x + self._out(self._attn(q, k, v, lambda r: keys[None] <= r[:, None]), p + "multihead_attn.")
            x = x + self._mlp(x, p)
        return rec

    def token_logp(self, ids: torch.Tensor, rec) -> torch.Tensor:
        """ids [T] one variant row -> [T - 1] log p(ids[t+1] | record, ids[<= t]), 0 where the target is the mask token."""
        ids = ids.to(self.device)
        T = len(ids)
        pos = torch.arange(T, device=self.device)
        own = torch.arange(T, device=self.device)
        x = self.w["token_embed.weight"][ids]
        for l in range(self.L):
            p = f"decoder.layers.{l}."
            q, k, v = self._qkv(self._ln(x, p + "norm1"), p + "self_attn.", pos)
            x = x + self._out(self._attn(q, k, v, lambda r: own[None] <= r[:, None]), p + "self_attn.")
            q, k, v = self._qkv(self._ln(x, p + "norm2"), p + "multihead_attn.", pos)
            Tm = rec[l][0].shape[0] if rec else 0
            if Tm:
                k, v = torch.cat([rec[l][0], k]), torch.cat([rec[l][1], v])
            allk = torch.arange(Tm + T, device=self.device)
            x = x + self._out(self._attn(q, k, v, lambda r: allk[None] <= (r[:, None] + Tm)), p + "multihead_attn.")
            x = x + self._mlp(x, p)
        if self.norm:
            x = self._ln(x, "norm")
        lp = torch.log_softmax(x @ self.w["linear.weight"].T + self.w["linear.bias"], dim=-1)
        tgt = ids[1:]
        out = lp[:-1].gather(1, tgt[:, None]).squeeze(1)
        return torch.where(tgt == MASK, torch.zeros_like(out), out)
