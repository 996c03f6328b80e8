"""Host-side driver of the H100 RITA scorer (reference: proteingym/baselines/rita/compute_fitness.py).

``calc_fitness`` (:13-42) scores a protein as the sum over its chunks of 1023 residues, and over each chunk read left to right and
reversed, of the MEAN log-probability of the tokens ``tokenizer.encode(p)[1:]`` given their prefixes. ``RitaScorer`` plans every
(protein, chunk, direction) token row with decoder.plan, computes each distinct row once (a chunk without a mutation is the wild
type's), and scores the rows through decoder.ArScorer: right-padded ragged batches and, for rows that share at least 128 leading tokens
with the wild type in the same chunk and direction, only their suffix after one wild-type pass (exact; include/pgscore.h).
"""
from __future__ import annotations

import json
import os

import numpy as np
import torch

from . import _lib
from .checkpoint import RitaConfig, rotary_tables
from .decoder import CONTEXT, ArScorer, chunks, plan  # noqa: F401 - chunks and plan stay part of this module's interface


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


class RitaScorer(ArScorer):
    def __init__(self, conf: RitaConfig, state: dict, inv_freq: torch.Tensor, tokenizer: RitaTokenizer, precision: str = "f16f8",
                 device: int = 0, max_rows: int = 0, context: int = CONTEXT):
        self.tok, self.context, self.conf = tokenizer, context, conf
        self.max_T = context + tokenizer.n_special  # longest token row one chunk can give
        desc = _lib.PgModelDesc(arch=_lib.PG_ARCH_RITA, layers=conf.layers, embed_dim=conf.embed_dim, heads=conf.heads, ffn_dim=conf.ffn_dim,
                                vocab=conf.vocab, max_positions=self.max_T, token_dropout=0, emb_ln_before=0,
                                precision=_lib.PRECISIONS[precision], device=device, max_rows=max_rows)
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
