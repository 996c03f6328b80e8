"""Host-side driver of the H100 Tranception scorer (reference: proteingym/baselines/tranception).

``TranceptionScorer.score_mutants`` mirrors ``TranceptionLMHeadModel.score_mutants`` (tranception/model_pytorch.py:878-928):
slice (``get_sequence_slices``, utils/scoring_utils.py:152-203), score every distinct slice left-to-right and on the reversed
string (``get_tranception_scores_mutated_sequences``, :77-150), divide by the full sequence length, subtract the wild type
scored in the same window, average the two directions, append the WT row. The forward + token log-likelihood runs in the
CUDA library through the shared decoder driver (decoder.ArScorer: ragged batches, retrieval fusion, wild-type prefix reuse); pandas is
used only for the same bookkeeping the reference does with it.
"""
from __future__ import annotations

import json
import math
import os

import numpy as np
import pandas as pd
import torch

from . import _lib
from .decoder import CHUNK_ROWS, ArScorer, Fusion, prefix_split, reuse_plan

VOCAB = ["[UNK]", "[CLS]", "[SEP]", "[PAD]", "[MASK]"] + list("ACDEFGHIKLMNPQRSTVWY")
TOK = {t: i for i, t in enumerate(VOCAB)}
CLS, SEP, PAD = 1, 2, 3
AA_vocab = "ACDEFGHIKLMNPQRSTVWY"


def alibi_slopes(heads: int):
    """Grouped ALiBi (model_pytorch.py:50-71): geometric slopes for heads/4 heads, the list repeated four times, so head h
    gets slopes[h mod (heads/4)] while its conv-kernel group is h div (heads/4)."""
    def geometric(n):
        start = 2 ** (-2 ** -(math.log2(n) - 3))
        return [start ** (i + 1) for i in range(n)]

    def plain(n):
        if math.log2(n).is_integer():
            return geometric(n)
        c = 2 ** math.floor(math.log2(n))
        return geometric(c) + plain(2 * c)[0::2][:n - c]
    return plain(heads // 4) * 4


def conv_taps(state: dict, layer: int, heads: int) -> torch.Tensor:
    """[3 (q,k,v) * 4 groups * 64 channels, 8]: look-back taps tap[o] (out[t] = bias + sum_o tap[o] * x[t-o]) and the bias in
    column 7. Group 0 is the identity; groups 1..3 carry the depthwise Conv1d(k=3,5,7, padding=k-1, truncated) weights
    (model_pytorch.py:73-88, :240-251): conv weight index j multiplies x[t-(k-1)+j], i.e. look-back o = k-1-j."""
    taps = torch.zeros(3, 4, 64, 8, dtype=torch.float32)
    taps[:, 0, :, 0] = 1.0
    for wi, nm in enumerate(("query", "key", "value")):
        for gi, k in enumerate((3, 5, 7)):
            w = state[f"h.{layer}.attn.{nm}_depthwiseconv.{gi}.conv.weight"].float()  # [hd, 1, k]
            b = state[f"h.{layer}.attn.{nm}_depthwiseconv.{gi}.conv.bias"].float()
            taps[wi, gi + 1, :, :k] = torch.flip(w[:, 0, :], dims=(1,))
            taps[wi, gi + 1, :, 7] = b
    return taps.reshape(3 * 4 * 64, 8).contiguous()


def load_tranception_checkpoint(folder: str):
    """HF checkpoint directory -> (config dict, state with the ``transformer.`` prefix stripped), as
    ``TranceptionLMHeadModel.from_pretrained`` would consume it (score_tranception_proteingym.py:79-100)."""
    cfg = json.load(open(os.path.join(folder, "config.json")))
    pbin = os.path.join(folder, "pytorch_model.bin")
    if os.path.exists(pbin):
        raw = torch.load(pbin, map_location="cpu", weights_only=True)
    else:
        from safetensors.torch import load_file
        raw = load_file(os.path.join(folder, "model.safetensors"))
    state = {}
    for k, v in raw.items():
        if k.endswith(".attn.bias") or k.endswith(".attn.masked_bias") or k == "transformer.alibi" or k == "lm_head.weight":
            continue  # causal-mask / alibi buffers and the tied output matrix
        state[k[len("transformer."):] if k.startswith("transformer.") else k] = v.float().contiguous()
    return cfg, state


def tokenize(seq: str) -> list:
    return [CLS] + [TOK.get(c, 0) for c in seq] + [SEP]


_LUT = None


def tokenize_batch(seqs, T: int):
    """``[CLS] s [SEP]`` for every string, right-padded with [PAD] to T columns -> (ids [n, T] int32, lens [n] int32).
    Same ids as ``tokenize`` (characters outside the vocabulary -> [UNK] = 0), built with one table lookup instead of a Python loop
    per residue."""
    global _LUT
    if _LUT is None:
        _LUT = np.zeros(256, dtype=np.int32)
        for ch, i in TOK.items():
            if len(ch) == 1:
                _LUT[ord(ch)] = i
    n = len(seqs)
    L = np.fromiter((len(s) for s in seqs), dtype=np.int64, count=n)
    ids = np.full((n, T), PAD, dtype=np.int32)
    if n == 0:
        return ids, np.zeros(0, dtype=np.int32)
    ids[:, 0] = CLS
    flat = _LUT[np.frombuffer("".join(seqs).encode("latin-1", errors="replace"), dtype=np.uint8)]
    rows = np.repeat(np.arange(n), L)
    cols = np.arange(int(L.sum())) - np.repeat(np.cumsum(L) - L, L) + 1
    ids[rows, cols] = flat
    ids[np.arange(n), L + 1] = SEP
    return ids, (L + 2).astype(np.int32)


def replace_ambiguous(seq: str) -> str:
    """encode_batch (model_pytorch.py:930-938): X/B/J/Z are replaced by a random compatible residue (np.random, unseeded)."""
    for ch, repl in (("X", AA_vocab), ("B", "DN"), ("J", "IL"), ("Z", "EQ")):
        if ch in seq:
            s = list(seq)
            pos = [i for i, c in enumerate(s) if c == ch]
            picks = np.random.choice(a=list(repl), size=len(pos), replace=True)
            for i, p in zip(pos, picks):
                s[i] = p
            seq = "".join(s)
    return seq


def prior_rows(prow, prow2, ws, we, msa_start, msa_end, flip, nonfocus=None):
    """Index arithmetic of the retrieval fusion for one sequence slice [ws, we) of the full protein (Tranception
    model_pytorch.py:811-830; TranceptEVE model_pytorch.py:1085-1133): fill ``prow`` (and ``prow2`` for the EVE table) with the prior
    row to mix into each predicted position, in the encoding pg_ar_fusion documents. Position a0+i of the slice takes row lo+i
    (left-to-right) or hi-1-i (``flip``: the slice of the prior is reversed with the sequence).

    ``nonfocus`` (bool per prior row, TranceptEVE with a focus-column threshold < 1): rows where the EVE prior is -inf. The reference
    finds them after fusion, converts their position ix back to protein coordinates as ix + ws — also for flipped sequences, where
    that is not the position's true coordinate — and re-fuses them with the MSA prior alone, taking row (ix + ws) - lo of the
    (possibly reversed) prior slice, or with nothing but the (1 - alpha) factor when ix + ws falls outside the MSA."""
    lo, hi = max(ws, msa_start), min(we, msa_end)
    if not (msa_start < we and msa_end > ws) or hi <= lo:
        return
    n = hi - lo
    a0 = max(0, we - msa_end) if flip else max(0, msa_start - ws)
    rows = np.arange(hi - 1, lo - 1, -1) if flip else np.arange(lo, hi)
    prow[a0:a0 + n] = rows
    if prow2 is None:
        return
    prow2[a0:a0 + n] = rows
    if nonfocus is None:
        return
    for i in np.nonzero(nonfocus[rows])[0]:
        ix = a0 + int(i)
        full = ix + ws
        prow2[ix] = -1
        if msa_start <= full < msa_end:
            k = full - lo
            prow[ix] = (hi - 1 - k) if flip else (lo + k)
        else:
            prow[ix] = -2


class TranceptionScorer(ArScorer):
    """Tranception on a pg_ar_* handle. Its token rows are residue strings, scored as ``[CLS] s [SEP]``."""

    def __init__(self, config: dict, state: dict, precision: str = "f16f8", device: int = 0, max_rows: int = 0):
        d, heads, layers = int(config["n_embd"]), int(config["n_head"]), int(config["n_layer"])
        ffn = int(config["n_inner"]) if config.get("n_inner") else 4 * d
        self.n_ctx = int(config.get("n_ctx", config.get("n_positions", 1024)))
        if abs(float(config.get("layer_norm_epsilon", 1e-5)) - 1e-5) > 1e-12:
            raise _lib.PgError("layer_norm_epsilon != 1e-5 is not supported")
        if config.get("activation_function", "squared_relu") != "squared_relu":
            raise _lib.PgError("only the squared_relu activation is supported")
        self.vocab = int(config.get("vocab_size", 25))
        self.config = config
        desc = _lib.PgModelDesc(arch=_lib.PG_ARCH_TRANCEPTION, layers=layers, embed_dim=d, heads=heads, ffn_dim=ffn, vocab=self.vocab,
                                max_positions=self.n_ctx, token_dropout=0, emb_ln_before=0, precision=_lib.PRECISIONS[precision],
                                device=device, max_rows=max_rows)
        tensors = {k: v for k, v in state.items() if "depthwiseconv" not in k}
        for l in range(layers):
            tensors[f"h.{l}.attn.conv_taps"] = conv_taps(state, l, heads)
        tensors["alibi_slopes"] = torch.tensor(alibi_slopes(heads), dtype=torch.float32).view(-1, 1)
        super().__init__(desc, tensors, device)

    def row_len(self, row) -> int:
        return len(row) + 2

    def row_ids(self, rows, idx, T: int, start: int = 0) -> np.ndarray:
        ids, _ = tokenize_batch([replace_ambiguous(rows[k]) for k in idx], T)
        return np.ascontiguousarray(ids[:, start:])

    def row_token(self, row, t: int) -> int:
        return TOK.get(row[t - 1], 0)  # token t of [CLS] s [SEP] is character t - 1

    def fusion(self, seqs, windows, flip, prior=None, alpha=0.6, msa_start=0, msa_end=None, prior2=None, beta=0.0, first_col=0,
               nonfocus_fallback=False):
        """The retrieval fusion of model_pytorch.py:806-830 (TranceptEVE: the three-way fusion, see ``prior_rows``) for the strings
        ``seqs`` scored in ``windows`` [(start, end)] of the full protein; None without a prior."""
        if prior is None:
            return None
        msa_end = prior.shape[0] if msa_end is None else msa_end
        nonfocus = None
        if prior2 is not None and nonfocus_fallback and beta > 0:  # rows whose EVE prior is -inf drag the fused value to -inf (:1118)
            nonfocus = np.asarray(prior2)[:, 5:].min(axis=1) == -np.inf

        def rows(k):
            prow = np.full(len(seqs[k]) + 2, -1, dtype=np.int32)
            prow2 = prow.copy() if prior2 is not None else None
            prior_rows(prow, prow2, windows[k][0], windows[k][1], msa_start, msa_end, flip, nonfocus)
            return prow, prow2

        def dev(a):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(self.device) if a is not None else None
        return Fusion(dev(prior), rows, float(alpha), dev(prior2), float(beta), int(first_col))

    # ------------------------------------------------------------------------------------------------------------
    def sequence_logprobs(self, seqs, prior=None, windows=None, flip=False, alpha=0.6, msa_start=0, msa_end=None, chunk_rows=CHUNK_ROWS,
                          prior2=None, beta=0.0, first_col=0, nonfocus_fallback=False, return_rows=False):
        """sum_t log p(tok_{t+1} | tok_<=t) of ``[CLS] s [SEP]`` for every string in ``seqs`` (float32 numpy).
        ``prior`` ([L_full, vocab] log-probabilities) with per-sequence ``windows`` [(start, end)] enables the retrieval
        fusion of model_pytorch.py:806-830; ``flip`` marks right-to-left scoring (the strings are already reversed).
        ``prior2`` / ``beta`` / ``first_col`` / ``nonfocus_fallback``: the TranceptEVE three-way fusion (see ``prior_rows``).
        ``return_rows``: also return, per sequence, the fused log-probabilities [len(s) + 1, vocab] of every predicted position."""
        # the reference tokenises with truncation=True, max_length=n_ctx (model_pytorch.py:930-938 -> scoring_utils.py:97-101): a
        # string longer than n_ctx - 2 residues (indel mode, sliding windows never produce one) is cut, [CLS] and [SEP] stay
        seqs = [s[:self.n_ctx - 2] for s in seqs]
        fusion = self.fusion(seqs, windows, flip, prior, alpha, msa_start, msa_end, prior2, beta, first_col, nonfocus_fallback)
        res = self.token_sums(seqs, fusion, return_rows, chunk_rows)
        return (res[0].astype(np.float32), res[1]) if return_rows else res.astype(np.float32)

    # ------------------------------------------------------------------------------------------------------------
    # Exact wild-type-prefix reuse (decoder.py). A mutant slice that has the same length as the wild type cut with the same window shares
    # every token before its first change with it; with the attention tile of 128 rows, all rows before start = 128 * (first changed
    # token // 128) are taken from ONE wild-type pass per window.
    def reuse_policy(self, strings, windows, wts):
        """Tranception's reuse policy for the strings of one direction, ``wts[i]`` the wild-type string scored in the same window as
        strings[i] (or None) -> (rows, row_windows, plain, groups) for ArScorer.reuse_sums: ``rows`` = the strings followed by one wild-type
        string per reused (wild type, window), the groups' partners. A string reuses its wild type when the two differ, have the same
        length of more than 126 residues and no X/B/J/Z (those are re-drawn at random per call). A window pays for its extra wild-type pass
        (T rows) only when its mutants skip clearly more rows than that (sum of starts >= 2 T); otherwise (e.g. proteins longer than the
        context, where every mutant has its own window) its strings run whole."""
        tile = self.PREFIX_TILE
        key, start, saved = [None] * len(strings), [0] * len(strings), {}
        for i, (x, w) in enumerate(zip(strings, wts)):
            if (self.prefix_reuse and w is not None and x != w and len(x) == len(w) and len(x) + 2 > tile
                    and not any(c in "XBJZ" for c in x) and not any(c in "XBJZ" for c in w)):
                s = prefix_split(x, w, 1, tile)[1]          # token index of the first change is 1 + diff ([CLS] is token 0)
                if s:
                    key[i], start[i] = (w, windows[i]), s
                    saved[key[i]] = saved.get(key[i], 0) + s
        kept = [k for k, rows in saved.items() if rows >= 2 * (len(k[0]) + 2)]
        partner = {k: len(strings) + j for j, k in enumerate(kept)}
        start = [s if key[i] in partner else 0 for i, s in enumerate(start)]
        plain, groups = reuse_plan(range(len(strings)), [partner.get(k) for k in key], start)
        return list(strings) + [k[0] for k in kept], list(windows) + [k[1] for k in kept], plain, groups

    def _logprobs_with_reuse(self, strings, windows, wts, flip, prior_kw):
        """``sequence_logprobs(strings, windows=windows, flip=flip, **prior_kw)`` with wild-type prefix reuse (``reuse_policy``); the strings
        that run whole go through sequence_logprobs."""
        rows, row_windows, plain, groups = self.reuse_policy(strings, windows, wts)
        fusion = self.fusion(rows, row_windows, flip, **prior_kw) if groups else None

        def plain_sums(idx):
            return self.sequence_logprobs([strings[i] for i in idx], windows=[windows[i] for i in idx], flip=flip, **prior_kw)
        out = self.reuse_sums(rows, range(len(strings)), plain, groups, fusion, plain_sums)
        return out[:len(strings)].astype(np.float32)

    # ------------------------------------------------------------------------------------------------------------
    @staticmethod
    def _window(pos, L, W):
        half = W // 2
        if L <= W:
            return 0, L
        if pos < half:
            return 0, W
        if pos >= L - half:
            return L - W, L
        return max(0, pos - half), min(L, pos + half)

    def slices(self, df, target_seq, scoring_window="optimal", indel_mode=False, start_idx=1) -> pd.DataFrame:
        """Rows (mutated_sequence, sliced_mutated_sequence, window_start, window_end): every mutant's window followed by the
        wild type cut with the same window, de-duplicated in first-seen order (scoring_utils.py:152-203)."""
        ctx = self.n_ctx - 2
        L = len(target_seq)
        mseqs = list(df["mutated_sequence"])
        recs = []
        if scoring_window == "optimal":
            spans = []
            for mut, ms in zip(df["mutant"], mseqs):
                if indel_mode:
                    spans.append((0, len(ms)))
                else:
                    centre = int(np.array([int(m[1:-1]) - start_idx for m in mut.split(":")]).mean())
                    spans.append(self._window(centre, L, ctx))
            recs += [(ms, ms[a:b], a, b) for ms, (a, b) in zip(mseqs, spans)]
            for a, b in spans:
                e = L if indel_mode else b
                recs.append((target_seq, target_seq[a:e], a, e))
        elif scoring_window == "sliding":
            for w in range(1 + int(L / ctx)):
                a = w * ctx
                recs += [(ms, ms[a:a + ctx], a, min(len(ms), a + ctx)) for ms in mseqs]
                recs += [(target_seq, target_seq[a:a + ctx], a, min(L, a + ctx)) for _ in mseqs]
        else:
            raise ValueError(scoring_window)
        out = pd.DataFrame(recs, columns=["mutated_sequence", "sliced_mutated_sequence", "window_start", "window_end"])
        return out.drop_duplicates().reset_index(drop=True)

    shard = None  # (rank, world) with an initialised torch.distributed group: split the sequence rows of each direction over the ranks

    def _sharded_logprobs(self, strings, windows, reverse, prior_kw, wts=None):
        """``sequence_logprobs`` over all ``strings``; with ``self.shard`` set, every rank scores a strided subset (rows are sorted
        by length inside sequence_logprobs, so a stride balances the padded work) and one all-gather completes the vector
        (SURVEY.md §8e: the mutant row is the unit for Tranception). A sequence's value does not depend on what it is batched with,
        so the result is the same for any world size."""
        if wts is None:
            wts = [None] * len(strings)
        if self.shard is None or self.shard[1] <= 1:
            return self._logprobs_with_reuse(strings, windows, wts, reverse, prior_kw)
        import torch.distributed as dist
        rank, world = self.shard
        n = len(strings)
        mine = list(range(rank, n, world))
        local = self._logprobs_with_reuse([strings[i] for i in mine], [windows[i] for i in mine], [wts[i] for i in mine], reverse, prior_kw)
        width = (n + world - 1) // world
        dev = self.device if dist.get_backend() == "nccl" else torch.device("cpu")
        buf = torch.zeros(width, dtype=torch.float32, device=dev)
        buf[:len(mine)] = torch.from_numpy(np.asarray(local, dtype=np.float32)).to(dev)
        parts = [torch.empty_like(buf) for _ in range(world)]
        dist.all_gather(parts, buf)
        out = np.zeros(n, dtype=np.float32)
        for r in range(world):
            idx = np.arange(r, n, world)
            out[idx] = parts[r][:len(idx)].cpu().numpy()
        return out

    def _direction(self, sl, target_seq, name, scoring_window, reverse, prior_kw):
        strings = [s[::-1] for s in sl["sliced_mutated_sequence"]] if reverse else list(sl["sliced_mutated_sequence"])
        windows = list(zip(sl["window_start"], sl["window_end"]))
        sc = sl.copy()
        # wild type cut with the same window, in scoring direction (None when the slice has no such partner, e.g. sliding windows)
        wt_by_win = {(a, b): (x[::-1] if reverse else x) for ms, x, a, b in zip(sl["mutated_sequence"], sl["sliced_mutated_sequence"],
                                                                                sl["window_start"], sl["window_end"]) if ms == target_seq}
        wts = [None if ms == target_seq or scoring_window != "optimal" else wt_by_win.get((a, b))
               for ms, a, b in zip(sl["mutated_sequence"], sl["window_start"], sl["window_end"])]
        sc["score"] = self._sharded_logprobs(strings, windows, reverse, prior_kw, wts).astype(np.float32)
        if scoring_window == "sliding":
            sc = sc[["mutated_sequence", "score"]].groupby("mutated_sequence").sum().reset_index()
        sc["score"] = sc["score"] / sc["mutated_sequence"].map(len)
        is_wt = sc.mutated_sequence == target_seq
        mut, wt = sc[~is_wt], sc[is_wt]
        if scoring_window == "optimal":
            d = pd.merge(mut, wt, how="left", on=["window_start"], suffixes=("", "_wt"))
            d[name] = d["score"] - d["score_wt"]
        else:
            d = mut.copy()
            d[name] = d["score"] - list(wt["score"])[0]
        return d[["mutated_sequence", name]]

    def score_mutants(self, DMS_data: pd.DataFrame, target_seq: str, scoring_mirror=True, indel_mode=False, scoring_window="optimal",
                      log_prior=None, retrieval_inference_weight=0.6, MSA_start=0, MSA_end=None) -> pd.DataFrame:
        df = DMS_data.copy()
        if "mutated_sequence" not in df and not indel_mode:
            df["mutated_sequence"] = df["mutant"].apply(lambda m: apply_substitutions(target_seq, m))
        assert "mutated_sequence" in df, "DMS file to score does not have mutated_sequence column"
        if "mutant" not in df:
            df["mutant"] = df["mutated_sequence"]
        df = df[["mutated_sequence", "mutant"]].reset_index(drop=True)
        sl = self.slices(df, target_seq, scoring_window, indel_mode)
        pk = dict(prior=log_prior, alpha=retrieval_inference_weight, msa_start=MSA_start, msa_end=MSA_end) if log_prior is not None else {}
        print("Scoring sequences from left to right")
        out = self._direction(sl, target_seq, "avg_score_L_to_R", scoring_window, False, pk)
        if scoring_mirror:
            print("Scoring sequences from right to left")
            rl = self._direction(sl, target_seq, "avg_score_R_to_L", scoring_window, True, pk)
            out = pd.merge(out, rl, on="mutated_sequence", how="left", suffixes=("", "_R_to_L"))
            out["avg_score"] = (out["avg_score_L_to_R"] + out["avg_score_R_to_L"]) / 2.0
        else:
            out["avg_score"] = out["avg_score_L_to_R"]
        col = "mutant" if indel_mode else "mutated_sequence"
        if target_seq in DMS_data[col].values:  # WT row scores 0 by definition (model_pytorch.py:917-927)
            cols = [col, "avg_score_L_to_R", "avg_score_R_to_L", "avg_score"] if scoring_mirror else [col, "avg_score_L_to_R", "avg_score"]
            out = pd.concat([out, pd.DataFrame([[target_seq] + [0] * (len(cols) - 1)], columns=cols)], ignore_index=True)
        return out


def apply_substitutions(focus_seq: str, mutant: str, start_idx: int = 1) -> str:
    """scoring_utils.get_mutated_sequence (:16-31), same assertion messages."""
    s = list(focus_seq)
    for m in mutant.split(":"):
        f, pos, t = m[0], int(m[1:-1]), m[-1]
        rel = pos - start_idx
        assert f == focus_seq[rel], "Invalid from_AA or mutant position: " + str(m) + " from_AA: " + str(f) + " relative pos: " + str(rel) + " focus_seq: " + str(focus_seq)
        assert t in AA_vocab, "Mutant to_AA is invalid: " + str(m)
        s[rel] = t
    return "".join(s)
