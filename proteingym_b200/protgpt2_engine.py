"""Host-side driver of the H100 ProtGPT2 scorer (reference: proteingym/baselines/protgpt2/compute_fitness.py).

``calc_fitness`` (:13-43) cuts a protein into chunks of 1023 characters (RITA's chunking, decoder.chunks), and scores every chunk
read left to right and reversed by the MEAN log-probability of the tokens ``encode(p)[1:]`` given ``encode(p)[:-1]``; GPT-2's tokenizer
adds no special tokens. The protein's score is the sum over chunks and directions divided by 2 * n_chunks. ``Protgpt2Scorer`` plans every
distinct (chunk, direction) row once through decoder.plan and ArScorer's wild-type prefix reuse: the first differing TOKEN decides the
reusable prefix, which is exact for a causal decoder with absolute positions.
"""
from __future__ import annotations

import heapq
import json
import os

import numpy as np

from . import _lib
from .checkpoint import Protgpt2Config
from .decoder import CONTEXT, ArScorer, plan


class Protgpt2Tokenizer:
    """``AutoTokenizer.from_pretrained(dir).encode(p)`` of a GPT-2 byte-level BPE tokenizer, for strings of ASCII letters.

    Reads ``tokenizer.json`` or, without it, ``vocab.json`` + ``merges.txt`` (what GPT2TokenizerFast converts from). On a string of ASCII
    letters the GPT-2 pre-tokenizer regex yields one word and the byte-to-unicode map is the identity, so the ids are the BPE of the
    string's characters: merges applied lowest rank first, leftmost first among equal ranks, as the ``tokenizers`` library does. Anything
    else is refused with NotImplementedError rather than tokenised differently: other characters (spaces, digits, punctuation,
    non-ASCII), the text of a special token, and tokenizer features this encoder does not implement."""

    def __init__(self, folder: str):
        tj = os.path.join(folder, "tokenizer.json")
        self.added = []
        if os.path.isfile(tj):
            with open(tj) as fh:
                spec = json.load(fh)
            self._check(spec, tj)
            m = spec["model"]
            vocab, merges = m["vocab"], m["merges"]
            self.added = [a["content"] for a in spec.get("added_tokens", [])]
        else:
            with open(os.path.join(folder, "vocab.json")) as fh:
                vocab = json.load(fh)
            with open(os.path.join(folder, "merges.txt"), encoding="utf-8") as fh:
                merges = [ln.rstrip("\n") for ln in fh if ln.strip() and not ln.startswith("#version")]
            at = os.path.join(folder, "added_tokens.json")
            if os.path.isfile(at):
                with open(at) as fh:
                    self.added = list(json.load(fh))
        self.vocab = {t: int(i) for t, i in vocab.items()}
        self.ranks = {}
        for r, mg in enumerate(merges):
            a, b = mg.split(" ") if isinstance(mg, str) else mg
            self.ranks.setdefault((a, b), r)

    @staticmethod
    def _check(spec: dict, path: str):
        def refuse(what):
            raise NotImplementedError(f"{path}: {what} is not implemented by the ProtGPT2 tokenizer (GPT-2 byte-level BPE)")
        m = spec.get("model") or {}
        if m.get("type") != "BPE":
            refuse(f"model type {m.get('type')!r}")
        if m.get("dropout"):
            refuse("BPE dropout")
        if m.get("byte_fallback"):
            refuse("byte_fallback")
        if m.get("ignore_merges"):
            refuse("ignore_merges")
        if m.get("continuing_subword_prefix") or m.get("end_of_word_suffix"):
            refuse("a continuing-subword prefix or end-of-word suffix")
        if spec.get("normalizer") is not None:
            refuse(f"normalizer {spec['normalizer'].get('type')!r}")
        pt = spec.get("pre_tokenizer") or {}
        if pt.get("type") != "ByteLevel" or not pt.get("use_regex", True):
            refuse(f"pre-tokenizer {pt.get('type')!r} (not GPT-2's ByteLevel with its regex)")
        if pt.get("add_prefix_space"):
            refuse("add_prefix_space")
        pp = spec.get("post_processor")
        if pp is not None and pp.get("type") != "ByteLevel":
            refuse(f"post-processor {pp.get('type')!r} (it may add tokens)")

    def _bpe(self, word: str) -> list:
        syms = list(word)
        n = len(syms)
        nxt, prv, alive = list(range(1, n + 1)), list(range(-1, n - 1)), [True] * n
        nxt[-1] = -1
        heap = [(self.ranks[(syms[i], syms[i + 1])], i, syms[i], syms[i + 1]) for i in range(n - 1) if (syms[i], syms[i + 1]) in self.ranks]
        heapq.heapify(heap)
        while heap:
            _, i, a, b = heapq.heappop(heap)  # (rank, position of the left symbol): lowest rank, then leftmost
            j = nxt[i]
            if not alive[i] or syms[i] != a or j < 0 or syms[j] != b:
                continue  # stale: one side was merged since this pair was pushed
            syms[i] = a + b
            alive[j] = False
            nxt[i] = nxt[j]
            if nxt[j] >= 0:
                prv[nxt[j]] = i
            for l, r in ((prv[i], i), (i, nxt[i])):
                if l >= 0 and r >= 0 and (syms[l], syms[r]) in self.ranks:
                    heapq.heappush(heap, (self.ranks[(syms[l], syms[r])], l, syms[l], syms[r]))
        return [syms[i] for i in range(n) if alive[i]]

    def encode(self, p: str) -> list:
        if p and not (p.isascii() and p.isalpha()):
            raise NotImplementedError(f"{p[:40]!r}: only strings of ASCII letters are tokenised (the GPT-2 pre-tokenizer splits others)")
        for a in self.added:
            if a and a in p:
                raise NotImplementedError(f"sequence contains the special token {a!r}: added-token splitting is not implemented")
        if not p:
            return []
        try:
            return [self.vocab[s] for s in self._bpe(p)]
        except KeyError as e:
            raise NotImplementedError(f"symbol {e.args[0]!r} is not in the vocabulary") from None


class Protgpt2Scorer(ArScorer):
    def __init__(self, conf: Protgpt2Config, state: dict, tokenizer: Protgpt2Tokenizer, precision: str = "f16f8", device: int = 0,
                 max_rows: int = 0, context: int = CONTEXT):
        self.conf, self.tok, self.context = conf, tokenizer, context
        desc = _lib.PgModelDesc(arch=_lib.PG_ARCH_PROTGPT2, layers=conf.layers, embed_dim=conf.embed_dim, heads=conf.heads,
                                ffn_dim=conf.ffn_dim, vocab=conf.vocab, max_positions=conf.n_positions, token_dropout=0, emb_ln_before=0,
                                precision=_lib.PRECISIONS[precision], device=device, max_rows=max_rows)
        super().__init__(desc, state, device)

    def score(self, prots, wt: str | None = None) -> np.ndarray:
        """calc_fitness of every protein (float64): the mean target log-probability of every (chunk, direction), summed and divided by
        2 * n_chunks. ``wt``: the wild type, whose rows serve as prefixes for the mutants' rows in the same chunk and direction. Raises
        ValueError where the reference fails: a (chunk, direction) that encodes to fewer than two tokens. No token (an empty last chunk,
        L a multiple of 1023) gives a float tensor the embedding rejects; one token (a 1-character last chunk, or a chunk BPE merges
        into one token) gives an empty input that GPT2Model.forward cannot reshape (``input_ids.view(-1, 0)``)."""
        rows, index, wt_of = plan(prots, wt, self.context)
        toks = [self.tok.encode(s) for s in rows]
        needed = {r for idx in index for r in idx}
        short = [len(toks[r]) for r in needed if len(toks[r]) < 2]
        if short:
            raise ValueError(f"a chunk encodes to {min(short)} token(s), leaving no input to predict from: the reference's calc_fitness "
                             "fails on it too")
        if any(len(toks[r]) > self.conf.n_positions for r in needed):
            raise ValueError(f"a chunk encodes to more than n_positions = {self.conf.n_positions} tokens")
        sums = self.row_sums(toks, wt_of, needed)
        means = np.array([sums[r] / (len(t) - 1) if r in needed else 0.0 for r, t in enumerate(toks)], dtype=np.float64)
        return np.array([sum(float(means[r]) for r in idx) / len(idx) for idx in index], dtype=np.float64)
