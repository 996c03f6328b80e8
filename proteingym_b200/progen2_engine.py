"""Host-side driver of the H100 ProGen2 scorer (reference: proteingym/baselines/progen2/compute_fitness.py).

``calc_fitness`` (:34-86) cuts a protein into chunks of ``n_positions`` characters, and scores every chunk read left to right and
reversed by the MEAN log-probability of its targets ``ids[1:]`` given ``ids[:-1]``, taken over the 25 amino-acid logits 5..29 only; a
last target that is a terminal ('1' = 3 or '2' = 4) is dropped first. The protein's score is the sum over chunks and directions,
divided by 2 and by len(prot). ``Progen2Scorer`` plans every distinct (chunk, direction) row once, through RITA's planner and prefix
machinery (rita_engine.plan / ArScorer): a row that drops its last target is scored as the token row ids[:-1], which the causal
decoder computes identically.
"""
from __future__ import annotations

import numpy as np

from . import _lib
from .checkpoint import Progen2Config, progen2_rotary_tables
from .rita_engine import PRECISIONS, ArScorer, plan

FIRST_COL, LAST_COL = 5, 29  # compute_fitness.py:71: the scored logits
TERMINALS = (3, 4)           # '1' / '2' (:63)


class Progen2Tokenizer:
    """``Tokenizer.from_str(tokenizer.json).encode(p).ids`` for ProGen2's fixed tokenizer file: a ByteLevel pre-tokenizer (every UTF-8
    byte becomes one symbol; printable ASCII maps to itself) and a BPE model without merges or unknown token over
    <|pad|> <|bos|> <|eos|> 1 2 A..Z (no J), so every symbol outside that vocabulary is silently dropped. The special tokens'
    own strings, which the library would split out as ids 0..2, are refused with NotImplementedError."""
    VOCAB = {c: i for i, c in enumerate(["1", "2"] + [c for c in "ABCDEFGHIKLMNOPQRSTUVWXYZ"], start=3)}
    SPECIALS = ("<|pad|>", "<|bos|>", "<|eos|>")

    def encode(self, p: str) -> list:
        for s in self.SPECIALS:
            if s in p:
                raise NotImplementedError(f"sequence contains the special token {s!r}: added-token splitting is not implemented")
        return [self.VOCAB[chr(b)] for b in p.encode("utf-8") if chr(b) in self.VOCAB]


def target_row(ids: list):
    """One (chunk, direction) of calc_fitness (:55-78) -> (the token row to score, number of targets): ids[:-1] with the last token
    dropped when it is a terminal target. Raises ValueError where the reference fails: fewer than two tokens (an empty chunk gives
    a float tensor, one token an empty target list), or a terminal among the remaining targets (the asserts at :67-68)."""
    if len(ids) < 2:
        raise ValueError(f"a chunk encodes to {len(ids)} token(s): the reference's calc_fitness fails on it too")
    if ids[-1] in TERMINALS:
        ids = ids[:-1]
    if any(t in TERMINALS for t in ids[1:]):
        raise ValueError("a terminal ('1' / '2') among the targets: the reference's calc_fitness asserts (compute_fitness.py:67-68)")
    return ids, len(ids) - 1


class Progen2Scorer(ArScorer):
    def __init__(self, conf: Progen2Config, state: dict, precision: str = "f16f8", device: int = 0, max_rows: int = 0):
        self.conf, self.context, self.tok = conf, conf.n_positions, Progen2Tokenizer()
        slot = 64 if conf.head_dim == 64 else 128
        desc = _lib.PgModelDesc(arch=_lib.PG_ARCH_PROGEN2, layers=conf.layers, embed_dim=conf.embed_dim, heads=conf.heads,
                                ffn_dim=conf.ffn_dim, vocab=conf.vocab, max_positions=conf.n_positions, token_dropout=0, emb_ln_before=0,
                                precision=PRECISIONS[precision], device=device, max_rows=max_rows)
        tensors = dict(state)
        tensors["rotary.cos"], tensors["rotary.sin"] = progen2_rotary_tables(conf.rotary_dim, slot, conf.n_positions)
        super().__init__(desc, tensors, device, head_vocab=LAST_COL - FIRST_COL + 1, label_off=FIRST_COL)

    def score(self, prots, wt: str | None = None) -> np.ndarray:
        """calc_fitness(reduction='mean') of every protein (float64); NaN when a (chunk, direction) keeps no target (the reference's
        CrossEntropyLoss mean over zero targets). ``wt``: the wild type as scored (with its terminals if the mutants have them), whose
        rows serve as prefixes for the mutants' rows in the same chunk and direction. Raises ValueError where the reference fails."""
        rows, index, wt_of = plan(prots, wt, self.context)
        needed = {r for idx in index for r in idx}
        toks, ntg = [], np.zeros(len(rows))
        for r, s in enumerate(rows):
            ids = self.tok.encode(s)
            if r in needed:
                ids, ntg[r] = target_row(ids)
            toks.append(ids)
        sums = self.row_sums(toks, wt_of, needed)
        with np.errstate(invalid="ignore", divide="ignore"):
            means = np.where(ntg > 0, sums / np.maximum(ntg, 1), np.nan)
        return np.array([sum(float(means[r]) for r in idx) / 2.0 / len(p) for p, idx in zip(prots, index)], dtype=np.float64)
