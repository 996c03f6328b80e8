"""Host-side driver shared by the autoregressive scorers (Tranception, RITA, ProGen2, ProtGPT2): the (chunk, direction) row planner of
the RITA-style reference scripts, right-padded ragged batches through the three pg_ar_* calls, and exact wild-type prefix reuse.

Prefix reuse (include/pgscore.h: pg_ar_prefix_begin / pg_ar_loglik_prefix): in a causal decoder every hidden state of a row before its
first token that differs from a wild-type row equals the wild type's, so

    sum(row) = sum(wt rows 0 .. start-2) + lp_wt[start-1, row[start]] + sum(row's rows start ..)

with ``start`` the first differing token rounded down to the 128-row attention tile. One wild-type pass records every layer's keys and
values; its rows then only run their suffix. Which rows reuse which wild type (the policy) stays with each model; ``reuse_plan``
groups them and ``ArScorer.reuse_sums`` runs the groups, counting the token rows saved in ``reuse_rows``.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import os
from typing import Callable

import numpy as np
import torch

from . import _lib

CONTEXT = 1023          # the RITA / ProtGPT2 scripts' model_context_len
CHUNK_ROWS = 1 << 17    # padded token rows per pg_ar_* call


def chunks(prot: str, context: int = CONTEXT) -> list:
    """calc_fitness's chunking (RITA compute_fitness.py:20-29): one chunk below ``context`` residues, else 1 + int(L / context) chunks of
    ``context`` residues (the last one may be short or empty)."""
    if len(prot) < context:
        return [prot]
    return [prot[i * context:(i + 1) * context] for i in range(1 + int(len(prot) / context))]


def plan(prots, wt: str | None = None, context: int = CONTEXT):
    """-> (rows, index, wt_of): ``rows`` the distinct strings to score (chunk or reversed chunk, in first-seen order), ``index[m]`` the
    row index of every (chunk, direction) of protein m in calc_fitness's summation order, ``wt_of[r]`` the row of the wild type's string
    in the same chunk and direction (None if there is no wild type, it is that row itself, or the lengths differ)."""
    rows, pos, index = [], {}, []

    def row(s):
        if s not in pos:
            pos[s] = len(rows)
            rows.append(s)
        return pos[s]
    wt_rows = {}
    if wt is not None:
        for k, c in enumerate(chunks(wt, context)):
            wt_rows[(k, 0)] = row(c)
            wt_rows[(k, 1)] = row(c[::-1])
    wt_of = {}
    for p in prots:
        idx = []
        for k, c in enumerate(chunks(p, context)):
            for dr, s in enumerate((c, c[::-1])):
                r = row(s)
                w = wt_rows.get((k, dr))
                if w is not None and w != r and len(rows[w]) == len(s):
                    wt_of.setdefault(r, w)
                idx.append(r)
        index.append(idx)
    return rows, index, wt_of


def prefix_split(x, w, offset: int = 1, tile: int = 128):
    """For a sequence ``x`` and the wild type ``w`` it shares a prefix with (both strings or token lists, in scoring order) -> (fd, start):
    fd = the token index of the first difference (``offset`` tokens precede element 0, e.g. 1 for [CLS]) and start = fd rounded down to
    the attention tile, the first row the transformer has to run for ``x``."""
    diff = next((k for k, (c, e) in enumerate(zip(x, w)) if c != e), len(x))
    fd = offset + diff
    return fd, (fd // tile) * tile


def prefix_total(wt_csum, wt_rows, start: int, label: int, suffix_sum) -> np.float32:
    """A sequence's summed log-likelihood recombined from its suffix pass (rows >= start) and the wild type's pass: rows < start - 1
    predict shared tokens (``wt_csum[k]`` = sum of the wild type's rows 0 .. k-1), row start - 1 has the wild type's state but predicts
    the sequence's own token ``label`` (``wt_rows`` [T, vocab]: the wild type's log-probability rows)."""
    return np.float32(wt_csum[start - 1] + float(wt_rows[start - 1, label]) + float(suffix_sum))


def length_batches(lens, chunk_rows: int = CHUNK_ROWS):
    """Right-padded ragged batches: index arrays into ``lens`` (token rows per row), sorted by length (stable), each grown while its
    padded size (rows x its longest row) stays within ``chunk_rows``, and at least one row."""
    lens = np.asarray(lens, dtype=np.int64)
    order = np.argsort(lens, kind="stable")
    i = 0
    while i < len(order):
        j = i + 1
        while j < len(order) and (j - i + 1) * lens[order[j]] <= chunk_rows:
            j += 1
        yield order[i:j]
        i = j


def reuse_plan(rows, partner, start):
    """Pure host planning of prefix reuse for the token rows ``rows`` (indices, in order): ``partner[r]`` the row whose wild-type pass
    serves row r and ``start[r]`` its first recomputed token (0: row r runs whole) -> (plain, groups): the rows that run whole, in order,
    and {partner: {start: [rows]}} in first-seen order. A partner that is itself one of ``rows`` takes its sum from its wild-type pass."""
    groups, plain = {}, []
    for r in rows:
        if start[r] > 0:
            groups.setdefault(partner[r], {}).setdefault(start[r], []).append(r)
        else:
            plain.append(r)
    return [r for r in plain if r not in groups], groups


@dataclasses.dataclass
class Fusion:
    """Retrieval fusion of the head (pg_ar_fusion in include/pgscore.h) for a list of token rows: the log-prior table(s) [L, vocab] on the
    device, their weights, and ``rows(k)`` -> (prow, prow2 or None), the prior-row vector(s) of token row k (int32, one entry per token;
    -1: no prior for that token). Batches pad them with -1."""
    prior: torch.Tensor
    rows: Callable
    alpha: float
    prior2: torch.Tensor | None = None
    beta: float = 0.0
    first_col: int = 0

    def take(self, idx):
        """The fusion of token rows ``idx`` of this one's."""
        return dataclasses.replace(self, rows=lambda k: self.rows(idx[k]))


class ArScorer(_lib.Model):
    """A pg_ar_* handle and the token-row machinery every autoregressive scorer shares: summed log-likelihoods of right-padded ragged
    token rows, optionally fused with retrieval priors, and wild-type prefix reuse. The head of the handle scores ``head_vocab`` token ids
    from ``label_off`` on (RITA: all of them; ProGen2: ids 5..29). Rows are token lists here; a subclass whose rows are something else
    (Tranception: residue strings) overrides ``row_len``, ``row_ids`` and ``row_token``."""
    prefix_reuse = os.environ.get("PG_PREFIX_REUSE", "1") != "0"
    PREFIX_TILE = 128
    PREFIX_MIN_TOKEN = 128  # RITA / ProGen2 / ProtGPT2: reuse a wild-type prefix when the first differing token is at least this far in
    reuse_rows = None       # [token rows a plain pass would run, token rows actually run], accumulated over calls (bench / tests)

    def __init__(self, desc, tensors: dict, device: int = 0, head_vocab: int = 0, label_off: int = 0):
        if desc.precision not in (_lib.PG_PREC_F16, _lib.PG_PREC_F16X3, _lib.PG_PREC_F16F8):
            raise KeyError("the autoregressive scorers take the precisions f16, f16x3 and f16f8 (f16d is built for the ESM masked marginals)")
        self.head_vocab, self.label_off = head_vocab or desc.vocab, label_off
        super().__init__(desc, tensors, device)

    def row_len(self, row) -> int:
        return len(row)

    def row_ids(self, rows, idx, T: int, start: int = 0) -> np.ndarray:
        """int32 [len(idx), T - start]: tokens start .. of rows ``idx``, right-padded."""
        ids = np.zeros((len(idx), T - start), dtype=np.int32)
        for r, k in enumerate(idx):
            ids[r, :len(rows[k]) - start] = rows[k][start:]
        return ids

    def row_token(self, row, t: int) -> int:
        return row[t]

    def _fusion(self, fusion, idx, T, start, keep, d_rows=None):
        """PgArFusion of one batch: rows ``idx`` of ``fusion`` from token ``start`` on, T columns; ``d_rows`` receives the rows."""
        f = _lib.PgArFusion(out_logprobs=d_rows.data_ptr() if d_rows is not None else None)
        if fusion is None:
            return f
        two = fusion.prior2 is not None
        prow = np.full((1 + two, len(idx), T), -1, dtype=np.int32)
        for r, k in enumerate(idx):
            for i, p in enumerate(fusion.rows(k)[:1 + two]):
                prow[i, r, :len(p) - start] = p[start:]
        keep.append(torch.from_numpy(prow).to(self.device))
        f.log_prior, f.prior_row, f.alpha, f.first_col = fusion.prior.data_ptr(), keep[-1][0].data_ptr(), fusion.alpha, fusion.first_col
        if two:
            f.log_prior2, f.prior_row2, f.beta = fusion.prior2.data_ptr(), keep[-1][1].data_ptr(), fusion.beta
        return f

    # ------------------------------------------------------------------------------------------------------------
    def token_sums(self, rows, fusion: Fusion | None = None, return_rows: bool = False, chunk_rows: int = CHUNK_ROWS):
        """sum_t log p(row[t+1] | row[<=t]) of every token row (float64 [n]; a row of fewer than two tokens scores 0), as right-padded
        ragged batches sorted by length through pg_ar_loglik_fused. ``return_rows``: also, per row, its (fused) log-probability rows
        [len - 1, head_vocab]."""
        out, rows_out = np.zeros(len(rows), dtype=np.float64), [None] * len(rows)
        lens = np.array([self.row_len(x) for x in rows], dtype=np.int64)
        scored = np.flatnonzero(lens >= 2)
        for idx in (scored[b] for b in length_batches(lens[scored], chunk_rows)):
            T = int(lens[idx[-1]])
            keep = []
            d_rows = torch.zeros((len(idx), T, self.head_vocab), dtype=torch.float32, device=self.device) if return_rows else None
            f = self._fusion(fusion, idx, T, 0, keep, d_rows)
            d_ids = torch.from_numpy(self.row_ids(rows, idx, T)).to(self.device)
            d_lens = torch.from_numpy(lens[idx].astype(np.int32)).to(self.device)
            d_out = torch.empty(len(idx), dtype=torch.float32, device=self.device)
            _lib.check(self.lib.pg_ar_loglik_fused(self.handle, d_ids.data_ptr(), d_lens.data_ptr(), len(idx), T, C.byref(f),
                                                   d_out.data_ptr(), self.stream()), self.handle)
            out[idx] = d_out.cpu().numpy()
            if return_rows:
                h_rows = d_rows.cpu().numpy()
                for r, k in enumerate(idx):
                    rows_out[k] = h_rows[r, :lens[k] - 1]
        return (out, rows_out) if return_rows else out

    def prefix_begin(self, row, fusion: Fusion | None = None):
        """Records the wild type ``row``'s keys / values -> (token log-probs [T], (fused) log-probability rows [T, head_vocab]) as numpy."""
        T = self.row_len(row)
        keep = []
        d_ids = torch.from_numpy(self.row_ids([row], [0], T)).to(self.device)
        d_tok = torch.zeros(T, dtype=torch.float32, device=self.device)
        d_rows = torch.zeros((T, self.head_vocab), dtype=torch.float32, device=self.device)
        f = self._fusion(fusion, [0], T, 0, keep, d_rows)
        _lib.check(self.lib.pg_ar_prefix_begin(self.handle, d_ids.data_ptr(), T, C.byref(f), d_tok.data_ptr(), self.stream()), self.handle)
        return d_tok.cpu().numpy(), d_rows.cpu().numpy()

    def prefix_suffix_sums(self, rows, start: int, fusion: Fusion | None = None, chunk_rows: int = CHUNK_ROWS) -> np.ndarray:
        """Suffix sums (rows >= start, float64) of token rows that share tokens 0 .. start-1 with the recorded wild type (any lengths)."""
        out = np.zeros(len(rows), dtype=np.float64)
        lens = np.array([self.row_len(x) - start for x in rows], dtype=np.int64)
        for idx in length_batches(lens, chunk_rows):
            T = int(lens[idx[-1]])
            keep = []
            f = self._fusion(fusion, idx, T, start, keep)
            d_ids = torch.from_numpy(self.row_ids(rows, idx, start + T, start)).to(self.device)
            d_lens = torch.from_numpy(lens[idx].astype(np.int32)).to(self.device)
            d_out = torch.empty(len(idx), dtype=torch.float32, device=self.device)
            _lib.check(self.lib.pg_ar_loglik_prefix(self.handle, d_ids.data_ptr(), d_lens.data_ptr(), len(idx), T, start, C.byref(f),
                                                    d_out.data_ptr(), self.stream()), self.handle)
            out[idx] = d_out.cpu().numpy()
        return out

    def reuse_sums(self, rows, scored, plain, groups, fusion: Fusion | None = None, plain_sums=None) -> np.ndarray:
        """Summed log-likelihoods (float64 [len(rows)]) of the token rows ``scored`` under a ``reuse_plan`` (plain, groups): ``plain``
        through ``plain_sums(plain)`` (default: token_sums), then per partner one wild-type pass and, per start, the suffix sums of its
        members, recombined with prefix_total. Adds the token rows of ``scored`` and those actually run to ``reuse_rows``."""
        out = np.zeros(len(rows), dtype=np.float64)
        lens = [self.row_len(x) for x in rows]
        run = sum(lens[r] for r in plain)
        if plain:
            out[plain] = plain_sums(plain) if plain_sums else self.token_sums([rows[r] for r in plain], fusion and fusion.take(plain))
        for w, by_start in groups.items():
            wt_tok, wt_rows = self.prefix_begin(rows[w], fusion and fusion.take([w]))
            run += lens[w]
            csum = np.concatenate([[0.0], np.cumsum(wt_tok.astype(np.float64))])    # csum[k] = sum of rows 0 .. k-1
            out[w] = csum[-1]
            for start, members in sorted(by_start.items()):
                sfx = self.prefix_suffix_sums([rows[r] for r in members], start, fusion and fusion.take(members))
                run += sum(lens[r] - start for r in members)
                for r, s in zip(members, sfx):
                    out[r] = prefix_total(csum, wt_rows, start, self.row_token(rows[r], start) - self.label_off, s)
        if self.reuse_rows is None:
            self.reuse_rows = [0, 0]
        self.reuse_rows[0] += sum(lens[r] for r in scored)
        self.reuse_rows[1] += run
        return out

    def row_sums(self, toks, wt_of, needed) -> np.ndarray:
        """Summed token log-likelihood of the planned token rows in ``needed`` (others: 0); rows with a wild-type partner ``wt_of[r]``
        whose first differing token is at least PREFIX_MIN_TOKEN in run as suffixes after one wild-type pass per partner, which also gives
        the partner's own sum."""
        scored = sorted(needed)
        start = dict.fromkeys(scored, 0)
        for r in scored:
            w = wt_of.get(r)
            if self.prefix_reuse and w is not None:
                fd, s = prefix_split(toks[r], toks[w], 0, self.PREFIX_TILE)
                if fd >= self.PREFIX_MIN_TOKEN and s < len(toks[r]) and s < len(toks[w]):
                    start[r] = s
        return self.reuse_sums(toks, scored, *reuse_plan(scored, wt_of, start))
