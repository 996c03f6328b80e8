"""Host-side driver of the H100 Tranception scorer (reference: proteingym/baselines/tranception).

``TranceptionScorer.score_mutants`` mirrors ``TranceptionLMHeadModel.score_mutants`` (tranception/model_pytorch.py:878-928):
slice (``get_sequence_slices``, utils/scoring_utils.py:152-203), score every distinct slice left-to-right and on the reversed
string (``get_tranception_scores_mutated_sequences``, :77-150), divide by the full sequence length, subtract the wild type
scored in the same window, average the two directions, append the WT row. The forward + token log-likelihood runs in the
CUDA library (``pg_ar_loglik``); pandas is used only for the same bookkeeping the reference does with it.
"""
from __future__ import annotations

import ctypes as C
import json
import math
import os

import numpy as np
import pandas as pd
import torch

from . import _lib

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


def prefix_split(x, w, offset: int = 1, tile: int = 128):
    """Exact wild-type-prefix reuse in a causal decoder: for a sequence ``x`` and the wild type ``w`` it shares a prefix with (both strings
    or token lists, in scoring order) -> (fd, start): fd = the token index of the first difference (``offset`` tokens precede element 0,
    e.g. 1 for [CLS]) and start = fd rounded down to the attention tile, the first row the transformer has to run for ``x``."""
    diff = next((k for k, (c, e) in enumerate(zip(x, w)) if c != e), len(x))
    fd = offset + diff
    return fd, (fd // tile) * tile


def prefix_total(wt_csum, wt_rows, start: int, label: int, suffix_sum) -> np.float32:
    """A sequence's summed log-likelihood recombined from its suffix pass (rows >= start) and the wild type's pass: rows < start - 1
    predict shared tokens (``wt_csum[k]`` = sum of the wild type's rows 0 .. k-1), row start - 1 has the wild type's state but predicts
    the sequence's own token ``label`` (``wt_rows`` [T, vocab]: the wild type's log-probability rows)."""
    return np.float32(wt_csum[start - 1] + float(wt_rows[start - 1, label]) + float(suffix_sum))


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


class TranceptionScorer:
    def __init__(self, config: dict, state: dict, precision: str = "f16f8", device: int = 0, max_rows: int = 0):
        if not torch.cuda.is_available():
            raise _lib.PgError("no CUDA device: the H100 scorer has no CPU fallback")
        self.lib = _lib.load()
        self.device = torch.device("cuda", device)
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
                                max_positions=self.n_ctx, token_dropout=0, emb_ln_before=0,
                                precision={"f16": _lib.PG_PREC_F16, "f16x3": _lib.PG_PREC_F16X3, "f16f8": _lib.PG_PREC_F16F8}[precision], device=device,
                                max_rows=max_rows)
        self.handle = C.c_void_p()
        _lib.check(self.lib.pg_create(C.byref(desc), C.byref(self.handle)))
        try:
            tensors = {k: v for k, v in state.items() if "depthwiseconv" not in k}
            for l in range(layers):
                tensors[f"h.{l}.attn.conv_taps"] = conv_taps(state, l, heads)
            tensors["alibi_slopes"] = torch.tensor(alibi_slopes(heads), dtype=torch.float32).view(-1, 1)
            gpu = [(n, t.to(self.device, torch.float32).contiguous()) for n, t in tensors.items()]
            arr = (_lib.PgTensor * len(gpu))()
            for i, (n, t) in enumerate(gpu):
                arr[i].name = n.encode()
                arr[i].data = t.data_ptr()
                arr[i].shape[0] = t.shape[0]
                arr[i].shape[1] = t.shape[1] if t.dim() == 2 else 1
            torch.cuda.synchronize(self.device)
            _lib.check(self.lib.pg_load_weights(self.handle, arr, len(gpu)), self.handle)
            del gpu
        except Exception:
            self.close()
            raise

    def close(self):
        if getattr(self, "handle", None) is not None and self.handle:
            self.lib.pg_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------------------------------------------------
    def sequence_logprobs(self, seqs, prior=None, windows=None, flip=False, alpha=0.6, msa_start=0, msa_end=None, chunk_rows=1 << 17,
                          prior2=None, beta=0.0, first_col=0, nonfocus_fallback=False, return_rows=False):
        """sum_t log p(tok_{t+1} | tok_<=t) of ``[CLS] s [SEP]`` for every string in ``seqs`` (float32 numpy).
        ``prior`` ([L_full, vocab] log-probabilities) with per-sequence ``windows`` [(start, end)] enables the retrieval
        fusion of model_pytorch.py:806-830; ``flip`` marks right-to-left scoring (the strings are already reversed).
        ``prior2`` / ``beta`` / ``first_col`` / ``nonfocus_fallback``: the TranceptEVE three-way fusion (see ``prior_rows``).
        ``return_rows``: also return, per sequence, the fused log-probabilities [len(s) + 1, vocab] of every predicted position."""
        n = len(seqs)
        out = np.zeros(n, dtype=np.float32)
        rows_out = [None] * n
        if n == 0:
            return (out, rows_out) if return_rows else out
        # the reference tokenises with truncation=True, max_length=n_ctx (model_pytorch.py:930-938 -> scoring_utils.py:97-101): a
        # string longer than n_ctx - 2 residues (indel mode, sliding windows never produce one) is cut, [CLS] and [SEP] stay
        seqs = [s[:self.n_ctx - 2] for s in seqs]
        order = np.argsort([len(s) for s in seqs], kind="stable")

        def dev32(a):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(self.device) if a is not None else None

        d_prior, d_prior2 = dev32(prior), dev32(prior2)
        msa_end = (prior.shape[0] if msa_end is None else msa_end) if prior is not None else None
        nonfocus = None
        if prior2 is not None and nonfocus_fallback and beta > 0:  # rows whose EVE prior is -inf drag the fused value to -inf (:1118)
            nonfocus = np.asarray(prior2)[:, 5:].min(axis=1) == -np.inf
        stream = torch.cuda.current_stream(self.device).cuda_stream
        i = 0
        while i < n:
            # grow the chunk while the padded row count stays within budget (sequences are sorted by length)
            j = i
            while j < n and (j - i + 1) * (len(seqs[order[j]]) + 2) <= chunk_rows:
                j += 1
            j = max(j, i + 1)
            idx = order[i:j]
            T = len(seqs[idx[-1]]) + 2
            ids, lens = tokenize_batch([replace_ambiguous(seqs[k]) for k in idx], T)
            prow = np.full((len(idx), T), -1, dtype=np.int32) if prior is not None else None
            prow2 = np.full((len(idx), T), -1, dtype=np.int32) if prior2 is not None else None
            if prior is not None:
                for r, k in enumerate(idx):
                    prior_rows(prow[r], prow2[r] if prow2 is not None else None, windows[k][0], windows[k][1], msa_start, msa_end, flip, nonfocus)
            d_ids = torch.from_numpy(ids).to(self.device)
            d_lens = torch.from_numpy(lens).to(self.device)
            d_prow = torch.from_numpy(prow).to(self.device) if prow is not None else None
            d_prow2 = torch.from_numpy(prow2).to(self.device) if prow2 is not None else None
            d_out = torch.empty(len(idx), dtype=torch.float32, device=self.device)
            d_rows = torch.zeros((len(idx), T, self.vocab), dtype=torch.float32, device=self.device) if return_rows else None
            f = _lib.PgArFusion(log_prior=d_prior.data_ptr() if d_prior is not None else None,
                                prior_row=d_prow.data_ptr() if d_prow is not None else None, alpha=float(alpha),
                                log_prior2=d_prior2.data_ptr() if d_prior2 is not None else None,
                                prior_row2=d_prow2.data_ptr() if d_prow2 is not None else None, beta=float(beta),
                                first_col=int(first_col), out_logprobs=d_rows.data_ptr() if d_rows is not None else None)
            _lib.check(self.lib.pg_ar_loglik_fused(self.handle, d_ids.data_ptr(), d_lens.data_ptr(), len(idx), T, C.byref(f),
                                                   d_out.data_ptr(), stream), self.handle)
            out[idx] = d_out.cpu().numpy()
            if return_rows:
                h_rows = d_rows.cpu().numpy()
                for r, k in enumerate(idx):
                    rows_out[k] = h_rows[r, :lens[r] - 1]
            i = j
        return (out, rows_out) if return_rows else out

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

    # ------------------------------------------------------------------------------------------------------------
    # Exact wild-type-prefix reuse (include/pgscore.h: pg_ar_prefix_begin / pg_ar_loglik_prefix). A mutant slice that has the same
    # length as the wild type cut with the same window shares every token before its first change with it; with the attention tile
    # of 128 rows, all rows before start = 128 * (first_changed_token // 128) are taken from ONE wild-type pass per window.
    prefix_reuse = os.environ.get("PG_PREFIX_REUSE", "1") != "0"
    PREFIX_TILE = 128
    reuse_rows = None  # [token rows a plain pass would run, token rows actually run], accumulated over calls (bench / tests)

    def _logprobs_with_reuse(self, strings, windows, wts, flip, prior_kw):
        """``sequence_logprobs(strings)`` where ``wts[i]`` is the wild-type string scored in the same window as strings[i] (or None).
        Strings eligible for reuse are grouped by (wild type, start) and scored as suffixes; the rest take the plain path."""
        n = len(strings)
        out = np.zeros(n, dtype=np.float32)
        tile = self.PREFIX_TILE
        groups, plain = {}, []
        for i, (x, w) in enumerate(zip(strings, wts)):
            start = 0
            if (self.prefix_reuse and w is not None and x != w and len(x) == len(w) and len(x) + 2 > tile
                    and not any(c in "XBJZ" for c in x) and not any(c in "XBJZ" for c in w)):  # those are re-drawn at random per call
                start = prefix_split(x, w, 1, tile)[1]          # token index of the first change is 1 + diff ([CLS] is token 0)
            if start > 0:
                groups.setdefault((w, windows[i], start), []).append(i)
            else:
                plain.append(i)
        by_wt = {}
        for (w, win, start), members in groups.items():
            by_wt.setdefault((w, win), []).append((start, members))
        # a window pays for its extra wild-type pass (T rows) only when its mutants skip clearly more rows than that; otherwise
        # (e.g. proteins longer than the context, where every mutant has its own window) its members take the plain path
        for key in list(by_wt):
            T = len(key[0]) + 2
            if sum(start * len(members) for start, members in by_wt[key]) < 2 * T:
                plain += [i for _, members in by_wt.pop(key) for i in members]
        plain.sort()
        rows_full = sum(len(x) + 2 for x in strings)
        rows_run = sum(len(strings[i]) + 2 for i in plain)
        if plain:
            out[plain] = self.sequence_logprobs([strings[i] for i in plain], windows=[windows[i] for i in plain], flip=flip, **prior_kw)
        for (w, win), lst in by_wt.items():
            rows_run += len(w) + 2
            wt_tok, wt_rows = self._prefix_begin(w, win, flip, prior_kw)
            csum = np.concatenate([[0.0], np.cumsum(wt_tok.astype(np.float64))])    # csum[k] = sum of rows 0 .. k-1
            for start, members in sorted(lst):
                rows_run += len(members) * (len(w) + 2 - start)
                suffix = self._prefix_suffix([strings[i] for i in members], win, start, flip, prior_kw)
                for i, sfx in zip(members, suffix):
                    tok_s = TOK.get(strings[i][start - 1], 0)                         # token `start` of [CLS] x [SEP] is character start-1
                    out[i] = prefix_total(csum, wt_rows, start, tok_s, sfx)
        if self.reuse_rows is None:
            self.reuse_rows = [0, 0]
        self.reuse_rows[0] += rows_full
        self.reuse_rows[1] += rows_run
        return out

    def _fusion(self, prior_kw, win, T, flip, n=1):
        """(PgArFusion, keep-alive tensors, prow, prow2) for ``n`` identical rows of T tokens in window ``win``."""
        prior, prior2 = prior_kw.get("prior"), prior_kw.get("prior2")
        keep = []
        if prior is None:
            return None, keep, None, None
        msa_start = prior_kw.get("msa_start", 0)
        msa_end = prior_kw.get("msa_end")
        msa_end = prior.shape[0] if msa_end is None else msa_end
        beta = prior_kw.get("beta", 0.0)
        nonfocus = None
        if prior2 is not None and prior_kw.get("nonfocus_fallback") and beta > 0:
            nonfocus = np.asarray(prior2)[:, 5:].min(axis=1) == -np.inf
        prow = np.full((T,), -1, dtype=np.int32)
        prow2 = np.full((T,), -1, dtype=np.int32) if prior2 is not None else None
        prior_rows(prow, prow2, win[0], win[1], msa_start, msa_end, flip, nonfocus)
        return (prior, prior2, beta), keep, prow, prow2

    def _prefix_begin(self, wt, win, flip, prior_kw):
        """Wild-type pass that records the prefix caches -> (token log-probs [T], fused rows [T, vocab]) as numpy."""
        T = len(wt) + 2
        ids, _ = tokenize_batch([replace_ambiguous(wt)], T)
        d_ids = torch.from_numpy(ids).to(self.device)
        meta, _, prow, prow2 = self._fusion(prior_kw, win, T, flip)
        d_tok = torch.zeros(T, dtype=torch.float32, device=self.device)
        d_rows = torch.zeros((T, self.vocab), dtype=torch.float32, device=self.device)
        f, keep = self._fusion_struct(meta, prow[None] if prow is not None else None, prow2[None] if prow2 is not None else None, prior_kw, d_rows)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.pg_ar_prefix_begin(self.handle, d_ids.data_ptr(), T, C.byref(f), d_tok.data_ptr(), stream), self.handle)
        return d_tok.cpu().numpy(), d_rows.cpu().numpy()

    def _fusion_struct(self, meta, prow, prow2, prior_kw, d_rows=None):
        keep = []

        def dev(a, dt):
            t = torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(self.device)
            keep.append(t)
            return t
        f = _lib.PgArFusion()
        f.alpha = float(prior_kw.get("alpha", 0.6))
        f.first_col = int(prior_kw.get("first_col", 0))
        if meta is not None:
            prior, prior2, beta = meta
            f.log_prior = dev(prior, np.float32).data_ptr()
            f.prior_row = dev(prow, np.int32).data_ptr()
            if prior2 is not None:
                f.log_prior2 = dev(prior2, np.float32).data_ptr()
                f.prior_row2 = dev(prow2, np.int32).data_ptr()
                f.beta = float(beta)
        if d_rows is not None:
            f.out_logprobs = d_rows.data_ptr()
        return f, keep

    def _prefix_suffix(self, seqs, win, start, flip, prior_kw, chunk_rows=1 << 17):
        """Suffix sums (rows >= start) of equal-length strings sharing tokens 0 .. start-1 with the recorded wild type."""
        T = len(seqs[0]) + 2
        Ts = T - start
        meta, _, prow, prow2 = self._fusion(prior_kw, win, T, flip)
        out = np.zeros(len(seqs), dtype=np.float32)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        per = max(1, chunk_rows // Ts)
        for i in range(0, len(seqs), per):
            part = seqs[i:i + per]
            ids, _ = tokenize_batch([replace_ambiguous(x) for x in part], T)
            d_ids = torch.from_numpy(np.ascontiguousarray(ids[:, start:])).to(self.device)
            d_lens = torch.full((len(part),), Ts, dtype=torch.int32, device=self.device)
            pr = np.repeat(prow[None, start:], len(part), axis=0) if prow is not None else None
            pr2 = np.repeat(prow2[None, start:], len(part), axis=0) if prow2 is not None else None
            f, keep = self._fusion_struct(meta, pr, pr2, prior_kw)
            d_out = torch.empty(len(part), dtype=torch.float32, device=self.device)
            _lib.check(self.lib.pg_ar_loglik_prefix(self.handle, d_ids.data_ptr(), d_lens.data_ptr(), len(part), Ts, start, C.byref(f),
                                                    d_out.data_ptr(), stream), self.handle)
            out[i:i + len(part)] = d_out.cpu().numpy()
        return out

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


def prefix_reuse_plan(slices: pd.DataFrame, target_seq: str, tile: int = 128) -> pd.DataFrame:
    """Planning aid for exact wild-type-prefix reuse (DESIGN.md §8.3; not used by the scorer yet). In a causal decoder every hidden
    state of a mutant before its first changed token equals the wild type's, so with the WT scored in the same window

        score(mutant) - score(WT) = [ lp_WT[fd-1, tok_m[fd]] - lp_WT[fd-1, tok_WT[fd]] ]            (row fd-1: same state, other label)
                                   + sum_{t >= fd} lp_m[t, label_m[t]] - sum_{t >= fd} lp_WT[t, label_WT[t]]

    where fd is the first token index at which the two ``[CLS] slice [SEP]`` strings differ and lp[t] the log-probability row that
    predicts token t+1. Only rows >= fd need the transformer (keys / values of earlier rows come from the WT run). For every
    (mutant slice, direction) this returns fd, the tile-aligned start the kernels would use, and the rows to compute, so the
    saving can be read off an assay before any kernel exists. ``slices``: output of ``TranceptionScorer.slices`` (optimal windows)."""
    wt_by_window = {(a, b): s for ms, s, a, b in zip(slices["mutated_sequence"], slices["sliced_mutated_sequence"], slices["window_start"],
                                                    slices["window_end"]) if ms == target_seq}
    recs = []
    for ms, s, a, b in zip(slices["mutated_sequence"], slices["sliced_mutated_sequence"], slices["window_start"], slices["window_end"]):
        if ms == target_seq:
            continue
        wt = wt_by_window.get((a, b))
        if wt is None or len(wt) != len(s):
            continue  # indels: no position-wise correspondence with a WT slice
        T = len(s) + 2
        for direction, x, y in (("L_to_R", s, wt), ("R_to_L", s[::-1], wt[::-1])):
            fd, start = prefix_split(x, y, 1, tile)          # token index ([CLS] is token 0)
            recs.append((ms, a, b, direction, T, fd, start, T - fd, T - start))
    return pd.DataFrame(recs, columns=["mutated_sequence", "window_start", "window_end", "direction", "tokens", "first_diff_token",
                                       "aligned_start", "rows_exact", "rows_tile_aligned"])


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
