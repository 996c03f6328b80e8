"""Cases and bounds of the Tranception fp64 tests (tests/test_gpu_tranception_fp64.py runs the kernels on them,
tests/test_tranception_fp64_bounds_cpu.py checks that the bounds would catch an emulated kernel fault on them).

Every case is a seeded synthetic model (``synth.make_tranception_state``, q/k gain 3) with ffn = 4 d and random proteins; the
reference is ``oracle.tranception_oracle.logprob_rows`` in fp64 on the same state, fused with the retrieval priors in fp64 where the
case has them."""
import functools
from dataclasses import dataclass

import numpy as np
import torch

from oracle import tranception_oracle as TO
from proteingym_b200 import synth
from proteingym_b200 import tranception_engine as TE

MODES = ["f16x3", "f16f8", "f16"]

# Max |log-prob - fp64 log-prob| over every predicted row and vocabulary column of every case below, per precision mode, measured on
# an H100 80GB HBM3 at a 700 W power limit (in the comments). The sums of the label columns are held to (tokens - 1) x the bound.
BOUND = {
    "f16x3": 8e-4,   # 4.1x the worst 1.94e-4 (h20-t1024; the fp32 oracle itself is ~1e-4 from fp64 at that width), typical 1e-4
    # 2.9x the worst 7.6e-4 (h20-l36-t1024; 7.1e-4 at two layers, h20-t1024), typical 6e-4. Not 4x: an attention that dropped P's
    # lo plane moves tokens by at most 4.9e-3 on this grid (tests/test_tranception_fp64_bounds_cpu.py), which 2x a 4x bound would miss
    "f16f8": 2.2e-3,
    "f16": 1e-1,     # 3.8x the worst 2.61e-2 (h16-t127), typical 2e-2
}

# tokens per sequence, [CLS] and [SEP] included: the empty protein; both sides of the 64-row attention / conv tiles; rows 64-69,
# whose conv look-back reads the previous conv tile's halo; both sides of the 128-row prefix tile; n_ctx (every key block, and
# the largest ALiBi term, slope 0.5 times key 1023 at 20 heads)
LENS = (2, 3, 63, 64, 65, 70, 71, 127, 128, 129, 1024)
RAGGED = (2, 3, 64, 65, 129, 300)
ALPHA, BETA = float(np.float32(0.6)), float(np.float32(0.3))  # the kernels mix with the fp32 weights


@functools.lru_cache(maxsize=None)
def model_state(layers, heads):
    d = 64 * heads
    return synth.make_tranception_state(synth.TranceptionArch(layers, d, heads, 4 * d), 100 * heads + layers)


@dataclass(frozen=True)
class Case:
    name: str
    heads: int
    lens: tuple                # tokens of each sequence scored in ONE sequence_logprobs call
    layers: int = 2
    fusion: int = 0            # 0: none; 2: retrieval prior (Tranception); 3: retrieval + EVE prior, first_col 5, flipped window
    cpu: bool = True           # part of the CPU fault sweep

    @property
    def id(self):
        return self.name

    @property
    def arch(self):
        d = 64 * self.heads
        return synth.TranceptionArch(self.layers, d, self.heads, 4 * d)

    def state(self):
        return model_state(self.layers, self.heads)

    def seqs(self):
        return [synth.random_protein(T - 2, 7 * T + self.heads) for T in self.lens]

    def fusion_inputs(self):
        """(sequence_logprobs keyword arguments, prow, prow2) of a fusion case: one sequence scored in window (0, L) of an
        L-residue protein. fusion 3: the window is scored flipped, the EVE prior is -inf on two row ranges (non-focus columns),
        so prow holds rows >= 0, -1 outside the MSA and -2 (non-focus, outside the MSA after the reference's unflipped
        index), and prow2 holds rows >= 0 and -1 (two-way fusion on the non-focus rows)."""
        L = self.lens[0] - 2
        rng = np.random.RandomState(self.heads + self.fusion)
        prior = np.log(rng.dirichlet(np.ones(25), size=L)).astype(np.float32)
        kw = dict(prior=prior, windows=[(0, L)], alpha=ALPHA, msa_start=40, msa_end=L - 30)
        if self.fusion == 3:
            prior2 = np.log(rng.dirichlet(np.ones(25), size=L)).astype(np.float32)
            prior2[150:160, 5:] = -np.inf  # flipped: positions >= msa_start, re-fused with the MSA prior alone
            prior2[210:220, 5:] = -np.inf  # flipped: positions < msa_start -> -2
            kw.update(prior2=prior2, beta=BETA, first_col=5, nonfocus_fallback=True, flip=True, msa_start=100, msa_end=250)
        prow = np.full(L + 2, -1, dtype=np.int32)
        prow2 = np.full(L + 2, -1, dtype=np.int32) if self.fusion == 3 else None
        nonfocus = np.asarray(kw["prior2"])[:, 5:].min(axis=1) == -np.inf if self.fusion == 3 else None
        TE.prior_rows(prow, prow2, 0, L, kw["msa_start"], kw["msa_end"], kw.get("flip", False), nonfocus)
        return kw, prow, prow2

    def reference(self, fault=None):
        """fp64 rows [len(s) + 1, V] per sequence (fused like pg_ar_fusion for a fusion case); ``fault``: one of TO.FAULTS."""
        rows = TO.logprob_rows(self.state(), self.seqs(), self.layers, self.heads, fault=fault)
        if self.fusion:
            kw, prow, prow2 = self.fusion_inputs()
            rows = [fuse(rows[0], prow, prow2, kw["prior"], kw.get("prior2"), kw.get("first_col", 0))]
        return rows

    def scorer(self, precision, max_rows=0):
        cfg = {"n_embd": self.arch.embed_dim, "n_head": self.heads, "n_layer": self.layers, "n_ctx": 1024, "n_inner": 4 * self.arch.embed_dim,
               "vocab_size": 25, "layer_norm_epsilon": 1e-5, "activation_function": "squared_relu"}
        st = {k[len("transformer."):]: v for k, v in self.state().items() if k.startswith("transformer.")}
        return TE.TranceptionScorer(cfg, st, precision=precision, max_rows=max_rows or 32768)

    def run(self, sc):
        """(sums [n] float32, rows [len(s) + 1, V] per sequence) of one sequence_logprobs call on the GPU."""
        kw = self.fusion_inputs()[0] if self.fusion else {}
        return sc.sequence_logprobs(self.seqs(), return_rows=True, **kw)


def fuse(lp, prow, prow2, prior, prior2, first_col):
    """pg_ar_fusion (include/pgscore.h) in fp64 on rows lp [n, V]: per row t and column v >= first_col, prow[t] >= 0 ->
    (1-alpha) lp + alpha prior[prow[t]], then (1-beta) . + beta prior2[prow2[t]] if prow2[t] >= 0; prow[t] == -2 -> (1-alpha) lp."""
    out = lp.copy()
    for t in range(lp.shape[0]):
        if prow[t] >= 0:
            m = (1 - ALPHA) * lp[t, first_col:] + ALPHA * prior[prow[t], first_col:].astype(np.float64)
            if prow2 is not None and prow2[t] >= 0:
                m = (1 - BETA) * m + BETA * prior2[prow2[t], first_col:].astype(np.float64)
            out[t, first_col:] = m
        elif prow[t] == -2:
            out[t, first_col:] = (1 - ALPHA) * lp[t, first_col:]
    return out


def label_sums(case, rows):
    """Sum over the predicted rows of each sequence of its next-token column."""
    out = []
    for s, r in zip(case.seqs(), rows):
        lab = TO.tokenize(s)[1:]
        out.append(float(np.asarray(r, dtype=np.float64)[np.arange(len(lab)), lab].sum()))
    return np.asarray(out)


def _grid():
    out = []
    for H in (4, 12, 16, 20):  # d 256 (one ALiBi slope, one head per conv group), the S, M and L head counts
        out += [Case(f"h{H}-t{T}", H, (T,)) for T in LENS]
        out.append(Case(f"h{H}-ragged", H, RAGGED))
    out += [Case("h12-fusion2", 12, (302,), fusion=2), Case("h12-fusion3", 12, (302,), fusion=3)]
    # Tranception-L depth (36 x 1280, 20 heads) at n_ctx
    out.append(Case("h20-l36-t1024", 20, (1024,), layers=36, cpu=False))
    return out


CASES = _grid()
BY_ID = {c.id: c for c in CASES}


def max_err(got, ref):
    return max(float(np.abs(np.asarray(g, dtype=np.float64) - r).max()) for g, r in zip(got, ref))

