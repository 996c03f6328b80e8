"""Window arithmetic for sequences longer than the model context (host side).
Reference: proteingym/utils/scoring_utils.py:43-52 (get_optimal_window), used at compute_fitness.py:492-495."""
from __future__ import annotations

import numpy as np


def optimal_window_starts(positions: np.ndarray, n_tokens: int, model_window: int = 1024):
    """Vectorised ``get_optimal_window``: for every masked token index return the start of its window and the common
    window length. Windows are ``[start, start + T)`` with ``T = min(n_tokens, model_window)``:
    left-aligned while the position is in the first half-window, right-aligned in the last half-window, centred
    (``pos - model_window // 2``) otherwise."""
    positions = np.asarray(positions, dtype=np.int64)
    if n_tokens <= model_window:
        return np.zeros(len(positions), dtype=np.int32), int(n_tokens)
    half = model_window // 2
    starts = positions - half
    starts = np.where(positions < half, 0, starts)
    starts = np.where(positions >= n_tokens - half, n_tokens - model_window, starts)
    return starts.astype(np.int32), int(model_window)


def esmc_window_starts(seq_positions: np.ndarray, seq_len: int, window_size: int = 1024):
    """ESM C's windows (evoscale compute_fitness.py:346-375), per 0-based residue index p: none while ``seq_len <= window_size - 2``;
    otherwise ``start = max(0, p - (window_size - 2) // 2)``, ``end = min(seq_len, start + window_size - 2)`` and, when ``end`` reaches
    the sequence end, ``start = max(0, seq_len - (window_size - 2))``. -> (residue starts int32, tokens per window incl. BOS/EOS)."""
    p = np.asarray(seq_positions, dtype=np.int64)
    span = window_size - 2
    if seq_len <= span:
        return np.zeros(len(p), dtype=np.int32), int(seq_len) + 2
    start = np.maximum(0, p - span // 2)
    end = np.minimum(seq_len, start + span)
    start = np.where(end == seq_len, max(0, seq_len - span), start)
    return start.astype(np.int32), int(window_size)


def esmc_window_rows(residue_tokens: np.ndarray, seq_positions: np.ndarray, cls_idx: int, eos_idx: int, window_size: int = 1024):
    """The token rows ESM C scores: each window re-tokenised as ``<cls> seq[start:end] <eos>`` (compute_fitness.py:377-394), one row
    per DISTINCT window, concatenated. -> (tokens int32 [rows * T], positions int32 [P] = row offset + index of residue p's token in
    its row, win_start int32 [P] = that row's offset, T)."""
    res = np.asarray(residue_tokens, dtype=np.int32)
    p = np.asarray(seq_positions, dtype=np.int64)
    starts, T = esmc_window_starts(p, len(res), window_size)
    uniq, row = np.unique(starts, return_inverse=True)
    tokens = np.concatenate([np.concatenate([[cls_idx], res[s:s + T - 2], [eos_idx]]) for s in uniq]) if len(uniq) else \
        np.concatenate([[cls_idx], res, [eos_idx]])
    offset = row.astype(np.int64) * T
    positions = offset + (p - starts) + 1
    return tokens.astype(np.int32), positions.astype(np.int32), offset.astype(np.int32), int(T)
