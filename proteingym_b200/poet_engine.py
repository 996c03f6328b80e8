"""PoET scoring (proteingym/baselines/PoET/scripts/score.py) on the H100.

Host side of PG_ARCH_POET: the Uniprot21 encoding (poet/alphabets.py), the a3m read, the NeighborsSampler weights with the O(N^2 L)
identity count in ``pg_msa_cluster_neighbors``, the sampler and the context build in numpy exactly as the reference draws them, and the
15-member ensemble (context lengths x max_similarity, each scored forward and on reversed arrays). Every context and variant row runs
through ``pg_poet_context`` / ``pg_poet_loglik``."""
from __future__ import annotations

import ctypes as C
import io
import itertools

import numpy as np
import torch

from proteingym_b200 import _lib

GAP, START, STOP, MASK = 20, 21, 22, 23
SIMILARITIES = [1.0, 0.95, 0.90, 0.70, 0.50]
THETA = 0.2
ZSTD_MAGIC = b"\x28\xb5\x2f\xfd"

_ENC = np.full(256, MASK, dtype=np.uint8)  # every byte outside the alphabet is the mask token (Alphabet(missing=mask))
for _i, _c in enumerate(b"ARNDCQEGHILKMFPSTWYV-*$X"):
    _ENC[_c] = _i
_ENC[ord("O")], _ENC[ord("U")] = 11, 4  # OUBZ synonyms; B and Z stay the mask token


def encode(s: bytes) -> np.ndarray:
    """Uniprot21(include_gap, include_startstop, distinct_startstop).encode."""
    return _ENC[np.frombuffer(s, dtype=np.uint8)]


def append_startstop(x: np.ndarray) -> np.ndarray:
    return np.concatenate([np.array([START], dtype=x.dtype), x, np.array([STOP], dtype=x.dtype)])


def read_maybe_zstd(path: str) -> bytes:
    """Bytes of an ``.a3m.zst`` file: decompressed with pyzstd or zstandard when it starts with the zstd magic, else taken as plain text."""
    data = open(path, "rb").read()
    if not data.startswith(ZSTD_MAGIC):
        return data
    try:
        import pyzstd
        return pyzstd.decompress(data)
    except ImportError:
        pass
    try:
        import zstandard
        return zstandard.ZstdDecompressor().decompressobj().decompress(data)
    except ImportError:
        raise RuntimeError(f"{path} is zstd-compressed: install the pyzstd or zstandard module to read it") from None


def parse_a3m(data: bytes) -> list[bytes]:
    """Sequences of a fasta-like file as poet/fasta.py parse_stream(upper=False) yields them: '#' lines skipped, lines stripped and joined."""
    seqs, cur, named = [], [], False
    for line in io.BytesIO(data):
        if line.startswith(b"#"):
            continue
        line = line.strip()
        if line.startswith(b">"):
            if named:
                seqs.append(b"".join(cur))
            named, cur = True, []
        else:
            cur.append(line)
    if named:
        seqs.append(b"".join(cur))
    return seqs


def weight_matrix(seqs: list[bytes]) -> np.ndarray:
    """The aligned matrix the weights are computed on: each row with its lower-case insertions deleted, encoded."""
    lower = bytes(range(ord("a"), ord("z") + 1))
    return np.vstack([encode(s.translate(None, delete=lower)) for s in seqs])


def context_sequence(s: bytes) -> bytes:
    """A sampled MSA row as it enters the context: upper-cased (insertions kept), gaps deleted."""
    return s.upper().translate(None, delete=b"-")


def min_matches(nongap: np.ndarray) -> np.ndarray:
    """Least m with the reference's float64 test ``1 - m / n <= theta`` (NeighborsSampler, theta 0.2), per row of n non-gap tokens."""
    out = np.empty(len(nongap), dtype=np.int32)
    cache = {}
    for i, n in enumerate(nongap.tolist()):
        if n not in cache:
            m = max(int(np.floor((1 - THETA) * n)) - 1, 0)
            while not (1 - np.float64(m) / np.float64(n) <= THETA):
                m += 1
            cache[n] = m
        out[i] = cache[n]
    return out


def neighbor_counts(msa: np.ndarray, device: int = 0) -> np.ndarray:
    """#{j : 1 - matches(i, j) / nongap(i) <= 0.2}, matches counted where both rows hold the same non-gap token (self included)."""
    nongap = (msa != GAP).sum(axis=1)
    if (nongap == 0).any():  # the reference divides 0 by 0 and fails its distance assertion
        raise AssertionError("an MSA row has no residue (all gaps): its identity to the other rows is undefined")
    tok = np.where(msa == GAP, 0, msa.astype(np.int32) + 1).astype(np.uint8)
    need = min_matches(nongap)
    dev = torch.device("cuda", device)
    d_tok = torch.from_numpy(np.ascontiguousarray(tok)).to(dev)
    d_need = torch.from_numpy(need).to(dev)
    d_out = torch.empty(len(tok), dtype=torch.int32, device=dev)
    lib = _lib.load()
    _lib.check(lib.pg_msa_cluster_neighbors(d_tok.data_ptr(), tok.shape[1], tok.shape[0], tok.shape[1], d_need.data_ptr(), d_out.data_ptr(),
                                            torch.cuda.current_stream(dev).cuda_stream))
    return d_out.cpu().numpy().astype(np.int64)


def sample_idxs(msa: np.ndarray, neighbors: np.ndarray, max_similarity: float, seed: int) -> np.ndarray:
    """MSASampler(NeighborsSampler, max_similarity).get_sample_idxs with the neighbour counts given."""
    p = 1 / neighbors
    p /= np.sum(p)
    norm_sim = (msa == msa[[0]]).sum(axis=1) / msa.shape[1]
    keep = np.where((norm_sim <= max_similarity) & (1 - norm_sim <= 1.0))[0]
    if len(keep) == 0:
        return np.array([], dtype=int)
    w = p[keep]
    rng = np.random.default_rng(seed)
    return keep[rng.choice(len(keep), replace=False, size=len(keep), p=w / w.sum())]


def sample_context(seqs: list[bytes], idxs: np.ndarray, max_tokens: int, seed: int) -> list[np.ndarray]:
    """sample_msa_sequences(truncate=False): sequences appended until the token total exceeds max_tokens (the last one overshoots),
    then shuffled by default_rng(seed).permutation."""
    out, total = [], 0
    for i in idxs:
        out.append(append_startstop(encode(context_sequence(seqs[i]))))
        total += len(out[-1])
        if total > max_tokens:
            break
    perm = np.random.default_rng(seed).permutation(len(out))
    final, total = [], 0
    for s in [out[i] for i in perm]:
        total += len(s)
        final.append(s)
        if total >= max_tokens:
            break
    return final


def reverse(rows: list[np.ndarray]) -> list[np.ndarray]:
    """The backward pass's arrays: every row reversed, so each starts with the stop token and ends with the start token."""
    return [np.ascontiguousarray(r[::-1]) for r in rows]


def rotary_tables(inv_freq: torch.Tensor, rows: int):
    """cos / sin [rows, 32] of the slot pairs (i, 32 + i): column i is the reference's frequency pair (2i, 2i + 1), fp32 as
    RotaryEmbedding.get_cos_sin_tables computes it."""
    f = torch.outer(torch.arange(rows).float(), inv_freq.float())[:, 0::2]
    return torch.cos(f).contiguous(), torch.sin(f).contiguous()


class PoetScorer(_lib.Model):
    """One PoET model on one device. ``max_positions``: the longest context sequence or variant row (tokens) a call may pass."""

    def __init__(self, conf, state: dict, max_positions: int, precision: str = "f16x3", device: int = 0, max_rows: int = 0):
        if precision not in ("f16", "f16x3", "f16f8"):
            raise ValueError(f"precision {precision!r}: PoET runs f16, f16x3 or f16f8")
        desc = _lib.PgModelDesc(arch=_lib.PG_ARCH_POET, layers=conf.layers, embed_dim=conf.hidden_dim, heads=conf.heads, ffn_dim=conf.ff_dim,
                                vocab=24, max_positions=max_positions, token_dropout=0, emb_ln_before=0,
                                precision=_lib.PRECISIONS[precision], device=device, max_rows=max_rows)
        tensors = {k: v for k, v in state.items() if not k.endswith("inv_freq")}
        tensors["rotary.cos"], tensors["rotary.sin"] = rotary_tables(state["rotary_emb.inv_freq"], max_positions)
        super().__init__(desc, tensors, device)
        self.d, self.np = conf.hidden_dim, 1 if precision == "f16" else 2
        self.mem_T = -1

    def set_context(self, rows: list[np.ndarray]):
        lens = (C.c_int32 * max(len(rows), 1))(*[len(r) for r in rows])
        ids = torch.from_numpy(np.concatenate(rows).astype(np.int32) if rows else np.zeros(1, np.int32)).to(self.device)
        _lib.check(self.lib.pg_poet_context(self.handle, ids.data_ptr(), lens, len(rows), self.stream()), self.handle)
        torch.cuda.synchronize(self.device)
        self.mem_T = sum(len(r) for r in rows)

    def record(self, layer: int):
        """(k, v) fp32 [mem_T, d] of the current context record at `layer`, in the reference's column order (rotated k)."""
        d = self.d
        raw = torch.empty((self.mem_T, 3 * d * self.np), dtype=torch.float16, device=self.device)
        _lib.check(self.lib.pg_poet_record(self.handle, layer, raw.data_ptr(), raw.stride(0) * 2, self.stream()), self.handle)
        torch.cuda.synchronize(self.device)
        full = raw[:, :3 * d].float() + (raw[:, 3 * d:].float() if self.np == 2 else 0)
        k, v = full[:, d:2 * d], full[:, 2 * d:]
        c = torch.arange(64)
        inv = torch.where(c % 2 == 0, c // 2, 32 + c // 2)  # reference dim c sits at slot inv[c]
        k = k.view(-1, d // 64, 64)[:, :, inv.to(self.device)].reshape(-1, d)
        return k, v

    def loglik(self, rows: list[np.ndarray], tok_logp: bool = False):
        """Σ log p(target) per row against the current context (targets = the mask token count 0); with tok_logp also [B, T] terms."""
        T = max(len(r) for r in rows)
        ids = np.full((len(rows), T), MASK, dtype=np.int32)
        for i, r in enumerate(rows):
            ids[i, :len(r)] = r
        d_ids = torch.from_numpy(ids).to(self.device)
        d_lens = torch.tensor([len(r) for r in rows], dtype=torch.int32, device=self.device)
        out = torch.empty(len(rows), dtype=torch.float32, device=self.device)
        tok = torch.empty((len(rows), T), dtype=torch.float32, device=self.device) if tok_logp else None
        _lib.check(self.lib.pg_poet_loglik(self.handle, d_ids.data_ptr(), d_lens.data_ptr(), len(rows), T, out.data_ptr(),
                                           tok.data_ptr() if tok is not None else None, self.stream()), self.handle)
        torch.cuda.synchronize(self.device)
        return (out.cpu().numpy(), tok.cpu().numpy()) if tok_logp else out.cpu().numpy()


def score_members(scorer: PoetScorer, msa_seqs: list[bytes], msa: np.ndarray, neighbors: np.ndarray, variants: list[np.ndarray],
                  context_lengths, seed: int) -> np.ndarray:
    """The ensemble of score.py main(): per (context length, max_similarity) the mean of the forward and backward scores, then the
    mean over members, in float32 as the reference's numpy arrays hold them."""
    logps = []
    for max_tokens, sim in itertools.product(context_lengths, SIMILARITIES):
        ctx = sample_context(msa_seqs, sample_idxs(msa, neighbors, sim, seed), max_tokens, seed)
        scorer.set_context(ctx)
        fwd = scorer.loglik(variants)
        scorer.set_context(reverse(ctx))
        bwd = scorer.loglik(reverse(variants))
        logps.append((fwd + bwd) / 2)
    return np.vstack(logps).mean(axis=0)
