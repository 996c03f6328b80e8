"""Host-side driver of the H100 RITA scorer (reference: proteingym/baselines/rita/compute_fitness.py).

``calc_fitness`` (:13-42) scores a protein as the sum over its chunks of 1023 residues, and over each chunk read left to right and
reversed, of the MEAN log-probability of the tokens ``tokenizer.encode(p)[1:]`` given their prefixes. ``RitaScorer`` plans every
(protein, chunk, direction) token row, computes each distinct row once (a chunk without a mutation is the wild type's), runs the rows
as right-padded ragged batches through ``pg_ar_loglik_fused`` and, for rows that share at least 128 leading tokens with the wild type
in the same chunk and direction, only their suffix through ``pg_ar_loglik_prefix`` (exact; include/pgscore.h).
"""
from __future__ import annotations

import ctypes as C
import json
import os

import numpy as np
import torch

from . import _lib
from .checkpoint import RitaConfig, rotary_tables
from .tranception_engine import prefix_split, prefix_total

CONTEXT = 1023  # calc_fitness's model_context_len


class RitaTokenizer:
    """``AutoTokenizer.from_pretrained(dir).encode(p)`` for a character-level ``tokenizer.json``: a BPE model without merges (every
    character is one vocabulary entry; a character outside it becomes the unknown token, or is dropped when the model has none, as the
    ``tokenizers`` library does), no normalizer, no pre-tokenizer, and no post-processor or a TemplateProcessing that wraps the sequence
    in special tokens. Any other tokenizer file is refused with NotImplementedError rather than tokenised differently."""

    def __init__(self, folder_or_file: str):
        path = os.path.join(folder_or_file, "tokenizer.json") if os.path.isdir(folder_or_file) else folder_or_file
        with open(path) as fh:
            spec = json.load(fh)
        m = spec.get("model") or {}

        def refuse(what):
            raise NotImplementedError(f"{path}: {what} is not implemented by the RITA tokenizer (character-level BPE without merges, "
                                      "no normalizer / pre-tokenizer, optional TemplateProcessing)")
        if m.get("type") != "BPE":
            refuse(f"model type {m.get('type')!r}")
        if m.get("merges"):
            refuse("a BPE model with merges")
        if m.get("dropout") or m.get("continuing_subword_prefix") or m.get("end_of_word_suffix") or m.get("fuse_unk") \
                or m.get("byte_fallback"):
            refuse("BPE dropout / subword prefix / word suffix / fuse_unk / byte_fallback")
        if spec.get("normalizer") is not None:
            refuse(f"normalizer {spec['normalizer'].get('type')!r}")
        if spec.get("pre_tokenizer") is not None:
            refuse(f"pre-tokenizer {spec['pre_tokenizer'].get('type')!r}")
        self.vocab = {t: int(i) for t, i in m["vocab"].items()}
        if any(len(t) != 1 for t in self.vocab if t not in {a["content"] for a in spec.get("added_tokens", [])}):
            refuse("a vocabulary entry longer than one character")
        self.unk = self.vocab.get(m["unk_token"]) if m.get("unk_token") else None
        self.added = [a["content"] for a in spec.get("added_tokens", [])]
        self.prefix, self.suffix = [], []
        pp = spec.get("post_processor")
        if pp is not None:
            if pp.get("type") != "TemplateProcessing":
                refuse(f"post-processor {pp.get('type')!r}")
            seen_a = False
            for item in pp["single"]:
                if "Sequence" in item:
                    if item["Sequence"]["id"] != "A" or seen_a:
                        refuse("a template other than specials + $A + specials")
                    seen_a = True
                else:
                    tok = item["SpecialToken"]["id"]
                    (self.suffix if seen_a else self.prefix).extend(int(i) for i in pp["special_tokens"][tok]["ids"])
            if not seen_a:
                refuse("a template without $A")

    @property
    def n_special(self) -> int:
        return len(self.prefix) + len(self.suffix)

    def encode(self, p: str) -> list:
        for a in self.added:
            if a in p:
                raise NotImplementedError(f"sequence contains the special token {a!r}: added-token splitting is not implemented")
        ids = []
        for c in p:
            i = self.vocab.get(c, self.unk)
            if i is not None:
                ids.append(i)
        return self.prefix + ids + self.suffix


def chunks(prot: str, context: int = CONTEXT) -> list:
    """calc_fitness's chunking (:20-29): one chunk below ``context`` residues, else 1 + int(L / context) chunks of ``context`` residues
    (the last one may be short or empty)."""
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


PRECISIONS = {"f16": _lib.PG_PREC_F16, "f16x3": _lib.PG_PREC_F16X3, "f16f8": _lib.PG_PREC_F16F8}


class ArScorer:
    """A pg_ar_* handle on the GPU and the token-row machinery every autoregressive scorer shares: summed log-likelihoods of ragged
    token rows, and wild-type prefix reuse for rows that share at least PREFIX_MIN_TOKEN leading tokens with a wild-type row. The head
    of the handle scores ``head_vocab`` token ids from ``label_off`` on (RITA: all of them; ProGen2: ids 5..29)."""
    prefix_reuse = os.environ.get("PG_PREFIX_REUSE", "1") != "0"
    PREFIX_TILE = 128
    PREFIX_MIN_TOKEN = 128  # reuse a wild-type prefix when the first differing token is at least this far in

    def __init__(self, desc, tensors: dict, device: int = 0, head_vocab: int = 0, label_off: int = 0):
        if not torch.cuda.is_available():
            raise _lib.PgError("no CUDA device: the H100 scorer has no CPU fallback")
        self.lib = _lib.load()
        self.device = torch.device("cuda", device)
        self.head_vocab, self.label_off = head_vocab or desc.vocab, label_off
        self.handle = C.c_void_p()
        _lib.check(self.lib.pg_create(C.byref(desc), C.byref(self.handle)))
        try:
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
        self.reuse_rows = [0, 0]  # token rows a plain pass would run, token rows actually run (accumulated; bench / tests)

    def close(self):
        if getattr(self, "handle", None) is not None and self.handle:
            self.lib.pg_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    # ------------------------------------------------------------------------------------------------------------
    def token_sums(self, ids_list, chunk_rows: int = 1 << 17) -> np.ndarray:
        """sum_t log p(ids[t+1] | ids[<=t]) of every token list (float64), as right-padded ragged batches sorted by length."""
        n = len(ids_list)
        out = np.zeros(n, dtype=np.float64)
        lens = np.array([len(x) for x in ids_list], dtype=np.int64)
        order = [i for i in np.argsort(lens, kind="stable") if lens[i] >= 2]
        i = 0
        while i < len(order):
            j = i
            while j < len(order) and (j - i + 1) * lens[order[j]] <= chunk_rows:
                j += 1
            j = max(j, i + 1)
            idx = order[i:j]
            T = int(lens[idx[-1]])
            ids = np.zeros((len(idx), T), dtype=np.int32)
            for r, k in enumerate(idx):
                ids[r, :lens[k]] = ids_list[k]
            d_ids = torch.from_numpy(ids).to(self.device)
            d_lens = torch.from_numpy(lens[idx].astype(np.int32)).to(self.device)
            d_out = torch.empty(len(idx), dtype=torch.float32, device=self.device)
            _lib.check(self.lib.pg_ar_loglik_fused(self.handle, d_ids.data_ptr(), d_lens.data_ptr(), len(idx), T, None, d_out.data_ptr(),
                                                   self._stream()), self.handle)
            out[idx] = d_out.cpu().numpy()
            i = j
        return out

    def prefix_begin(self, ids):
        """Records the wild type's keys / values -> (token log-probs [T], log-probability rows [T, vocab]) as numpy."""
        T = len(ids)
        d_ids = torch.tensor(ids, dtype=torch.int32, device=self.device)
        d_tok = torch.zeros(T, dtype=torch.float32, device=self.device)
        d_rows = torch.zeros((T, self.head_vocab), dtype=torch.float32, device=self.device)
        f = _lib.PgArFusion(out_logprobs=d_rows.data_ptr())
        _lib.check(self.lib.pg_ar_prefix_begin(self.handle, d_ids.data_ptr(), T, C.byref(f), d_tok.data_ptr(), self._stream()), self.handle)
        return d_tok.cpu().numpy(), d_rows.cpu().numpy()

    def prefix_suffix_sums(self, ids_list, start: int, chunk_rows: int = 1 << 17) -> np.ndarray:
        """Suffix sums (rows >= start) of token lists that share tokens 0 .. start-1 with the recorded wild type (any lengths)."""
        out = np.zeros(len(ids_list), dtype=np.float64)
        lens = np.array([len(x) - start for x in ids_list], dtype=np.int64)
        order = np.argsort(lens, kind="stable")
        i = 0
        while i < len(order):
            j = i
            while j < len(order) and (j - i + 1) * lens[order[j]] <= chunk_rows:
                j += 1
            j = max(j, i + 1)
            idx = order[i:j]
            T = int(lens[idx[-1]])
            ids = np.zeros((len(idx), T), dtype=np.int32)
            for r, k in enumerate(idx):
                ids[r, :lens[k]] = ids_list[k][start:]
            d_ids = torch.from_numpy(ids).to(self.device)
            d_lens = torch.from_numpy(lens[idx].astype(np.int32)).to(self.device)
            d_out = torch.empty(len(idx), dtype=torch.float32, device=self.device)
            _lib.check(self.lib.pg_ar_loglik_prefix(self.handle, d_ids.data_ptr(), d_lens.data_ptr(), len(idx), T, start, None,
                                                    d_out.data_ptr(), self._stream()), self.handle)
            out[idx] = d_out.cpu().numpy()
            i = j
        return out

    def row_sums(self, toks, wt_of, needed) -> np.ndarray:
        """Summed token log-likelihood of the planned token rows in ``needed`` (others: 0); rows with a wild-type partner whose first
        differing token is at least PREFIX_MIN_TOKEN in run as suffixes after one wild-type pass per partner, which also gives the
        partner's own sum."""
        n = len(toks)
        out = np.zeros(n, dtype=np.float64)
        groups, plain = {}, []
        for r, x in enumerate(toks):
            if r not in needed:
                continue
            w = wt_of.get(r)
            start = 0
            if self.prefix_reuse and w is not None:
                fd, start = prefix_split(x, toks[w], 0, self.PREFIX_TILE)
                if fd < self.PREFIX_MIN_TOKEN or start >= len(x) or start >= len(toks[w]):
                    start = 0
            if start > 0:
                groups.setdefault(w, {}).setdefault(start, []).append(r)
            else:
                plain.append(r)
        plain = [r for r in plain if r not in groups]
        self.reuse_rows[0] += sum(len(toks[r]) for r in needed)
        run = sum(len(toks[r]) for r in plain)
        if plain:
            out[plain] = self.token_sums([toks[r] for r in plain])
        for w, by_start in groups.items():
            wt_tok, wt_rows = self.prefix_begin(toks[w])
            run += len(toks[w])
            csum = np.concatenate([[0.0], np.cumsum(wt_tok.astype(np.float64))])
            out[w] = csum[-1]
            for start, members in sorted(by_start.items()):
                sfx = self.prefix_suffix_sums([toks[r] for r in members], start)
                run += sum(len(toks[r]) - start for r in members)
                for r, s in zip(members, sfx):
                    out[r] = float(prefix_total(csum, wt_rows, start, toks[r][start] - self.label_off, s))
        self.reuse_rows[1] += run
        return out


class RitaScorer(ArScorer):
    def __init__(self, conf: RitaConfig, state: dict, inv_freq: torch.Tensor, tokenizer: RitaTokenizer, precision: str = "f16f8",
                 device: int = 0, max_rows: int = 0, context: int = CONTEXT):
        self.tok, self.context, self.conf = tokenizer, context, conf
        self.max_T = context + tokenizer.n_special  # longest token row one chunk can give
        desc = _lib.PgModelDesc(arch=_lib.PG_ARCH_RITA, layers=conf.layers, embed_dim=conf.embed_dim, heads=conf.heads, ffn_dim=conf.ffn_dim,
                                vocab=conf.vocab, max_positions=self.max_T, token_dropout=0, emb_ln_before=0,
                                precision=PRECISIONS[precision], device=device, max_rows=max_rows)
        cos, sin = rotary_tables(inv_freq, self.max_T)
        tensors = dict(state)
        tensors["rotary.cos"], tensors["rotary.sin"] = cos, sin
        super().__init__(desc, tensors, device)

    def score(self, prots, wt: str | None = None) -> np.ndarray:
        """calc_fitness's score of every protein (float64): sum over (chunk, direction) of the mean target log-probability; NaN when a
        chunk leaves no target token (the reference's CrossEntropyLoss mean over zero targets). ``wt``: the wild type, whose rows serve
        as prefixes for the mutants' rows in the same chunk and direction. Raises ValueError where the reference fails: a chunk that
        encodes to no token at all."""
        rows, index, wt_of = plan(prots, wt, self.context)
        toks = [self.tok.encode(s) for s in rows]
        needed = {r for idx in index for r in idx}
        if any(not toks[r] for r in needed):  # torch.tensor([[]]) is a float tensor, which the reference's embedding rejects
            raise ValueError("a chunk encodes to no token (an empty last chunk, L a multiple of the context, with a tokenizer that adds "
                             "no special tokens): the reference's calc_fitness fails on it too")
        sums = self.row_sums(toks, wt_of, needed)
        ntg = np.array([len(t) - 1 for t in toks], dtype=np.float64)
        with np.errstate(invalid="ignore", divide="ignore"):
            means = np.where(ntg > 0, sums / np.maximum(ntg, 1), np.nan)
        return np.array([sum(float(means[r]) for r in idx) for idx in index], dtype=np.float64)
