"""Host-side driver of the H100 ProGen3 scorer (reference: proteingym/baselines/progen3/progen3/scorer.py, batch_preparer.py).

``ProGen3Scorer.score_batch`` (scorer.py:64-101) scores every sequence twice: N->C as ``<bos> 1 seq 2 <eos>`` and C->N as ``<bos>`` +
the reverse of ``1 seq 2`` + ``<eos>`` (batch_preparer.py:100-112), positions 0..T-1 and sequence ids 0. Each direction's score is the
mean fp32 cross entropy over its targets ``ids[1:]`` (no padding exists inside a row), negated; the sequence's log-likelihood is the
mean of the two directions and its perplexity exp(-ll). Batching does not change a score (right padding, causal attention), so rows run
through the shared decoder path (decoder.ArScorer) in whatever batches fit the workspace.
"""
from __future__ import annotations

import re

import numpy as np

from . import _lib
from .checkpoint import Progen3Config, progen3_rotary_tables
from .decoder import ArScorer

GLM_PATTERN = re.compile(r"^[A-Z]+\[GLM\](?:\d+\-\d+\-\d+;)*\d+\-\d+\-\d+;?$")  # batch_preparer.py:14
MAX_POSITIONS = 4096  # default rotary table rows: the longest ProteinGym protein (3 423 residues) plus its four added tokens fits


class Progen3Tokenizer:
    """``Tokenizer.from_file(tokenizer.json).encode(s).ids`` for ProGen3's fixed tokenizer: a ByteLevel pre-tokenizer and a BPE model
    without merges over <pad> <bos> <eos> <bos_glm> <eos_span> <mask> 1 2 A..Z (ids 0..33), so every other byte of the sequence is
    silently dropped. The special-token strings, which the library would split out, are only produced here around the sequence; inside
    it they are refused with NotImplementedError."""
    SPECIALS = ("<pad>", "<bos>", "<eos>", "<bos_glm>", "<eos_span>", "<mask>")
    VOCAB = {c: i for i, c in enumerate("12ABCDEFGHIJKLMNOPQRSTUVWXYZ", start=6)}
    PAD, BOS, EOS = 0, 1, 2

    def encode(self, seq: str, reverse: bool = False) -> list:
        """prepare_clm (batch_preparer.py:100-112): the token ids of one direction."""
        if "<" in seq and any(s in seq for s in self.SPECIALS) or "<span_" in seq:
            raise NotImplementedError("sequence contains a special-token string: added-token splitting is not implemented")
        s = "1" + seq + "2"
        if reverse:
            s = s[::-1]
        return [self.BOS] + [self.VOCAB[chr(b)] for b in s.encode("utf-8") if chr(b) in self.VOCAB] + [self.EOS]


def read_fasta(path: str) -> dict:
    """Bio.SeqIO.parse(path, "fasta") as scorer.run uses it (scorer.py:169-171): {record.id: sequence}. A record starts at a line beginning
    with '>'; its id is the first whitespace-separated token of the title (empty title: ""); its sequence is the following lines joined with
    spaces and carriage returns removed. Lines before the first record are skipped. A later record with the same id replaces the earlier."""
    seqs, cur, lines = {}, None, []
    with open(path) as fh:
        for line in fh:
            if line.startswith(">"):
                if cur is not None:
                    seqs[cur] = "".join(lines).replace(" ", "").replace("\r", "")
                title = line[1:].rstrip("\n").strip()
                cur, lines = (title.split(None, 1)[0] if title else ""), []
            elif cur is not None:
                lines.append(line.strip())
    if cur is not None:
        seqs[cur] = "".join(lines).replace(" ", "").replace("\r", "")
    return seqs


class Progen3Scorer(ArScorer):
    def __init__(self, conf: Progen3Config, state: dict, precision: str = "f16f8", device: int = 0, max_rows: int = 0,
                 max_positions: int = MAX_POSITIONS):
        self.conf, self.tok, self.max_positions = conf, Progen3Tokenizer(), max_positions
        desc = _lib.PgModelDesc(arch=_lib.PG_ARCH_PROGEN3, layers=conf.layers, embed_dim=conf.embed_dim, heads=conf.heads,
                                ffn_dim=conf.ffn_dim, vocab=conf.vocab, max_positions=max_positions, token_dropout=0, emb_ln_before=0,
                                precision=_lib.PRECISIONS[precision], device=device, max_rows=max_rows, kv_heads=conf.kv_heads,
                                n_experts=conf.n_experts, top_k=conf.top_k, gated_mlp=int(conf.gated_mlp), rms_eps=conf.rms_eps)
        tensors = dict(state)
        tensors["rotary.cos"], tensors["rotary.sin"] = progen3_rotary_tables(conf.head_dim, conf.rope_theta, max_positions)
        super().__init__(desc, tensors, device)

    def direction_scores(self, seqs) -> np.ndarray:
        """float64 [n, 2]: the N->C and C->N mean log-likelihoods (negated mean cross entropy) of every sequence."""
        for s in seqs:
            if GLM_PATTERN.match(s):
                raise NotImplementedError("GLM infilling inputs (batch_preparer.py:193) take another encoder, which is not implemented")
        rows = [self.tok.encode(s, rev) for s in seqs for rev in (False, True)]
        too_long = max(len(r) for r in rows) if rows else 0
        if too_long > self.max_positions:
            raise ValueError(f"a sequence encodes to {too_long} tokens, more than max_positions = {self.max_positions}")
        sums = self.token_sums(rows)
        ntg = np.array([len(r) - 1 for r in rows], dtype=np.float64)
        return (sums / ntg).reshape(len(seqs), 2)

    def score(self, seqs):
        """-> (log_likelihood, perplexity), float64 [n] each (scorer.py:64-76)."""
        d = self.direction_scores(list(seqs))
        ll = (d[:, 0] + d[:, 1]) / 2
        return ll, np.exp(-ll)
