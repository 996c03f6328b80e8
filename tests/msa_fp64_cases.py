"""Cases and bounds of the MSA Transformer fp64 tests (tests/test_gpu_z_msa_fp64.py runs the kernels on them,
tests/test_msa_fp64_bounds_cpu.py checks that the bounds would catch an emulated kernel fault on them).

Every case is a seeded synthetic model at q/k gain 1 (gain 2 makes the model ill-conditioned: DESIGN.md, MSA Transformer) and a
seeded random alignment; the reference is ``oracle.msa_oracle.masked_marginal_table`` in fp64 on the same state."""
from dataclasses import dataclass

import numpy as np
import torch

from oracle import msa_oracle as MO
from proteingym_b200 import checkpoint, msa_engine, synth

MODES = ["f16x3", "f16f8", "f16"]

# Max |log-prob - fp64 log-prob| over every case below, per precision mode: ~3.5-4x the worst value measured on an H100 80GB HBM3 at a
# 400 W power limit (in the comments; typical cases sit 2-5x lower still).
BOUND = {
    "f16x3": 4e-5,   # worst 1.14e-5 (h12; the fp32 oracle itself is 6.9e-6 from fp64 there), next 7.8e-6 (r130-row-only)
    "f16f8": 2e-4,   # worst 5.7e-5 (r1-column-only, h12), typical 3e-5
    "f16": 1e-2,     # worst 2.6e-3 (h12), typical 1e-3
}

# ablated states: the two attentions are told apart by zeroing the other one's output projection in every layer
STATES = ("full", "row-only", "column-only")


@dataclass(frozen=True)
class Case:
    name: str
    layers: int = 2
    d: int = 128
    heads: int = 2
    R: int = 5
    C: int = 41                   # alignment columns, BOS included
    positions: tuple = ()         # default: 0 (BOS), 1, an interior column and the last column
    per_pass: int = 0             # alignments per pass (0: up to 4)
    msa_pos_dim: int = 0
    embed_positions_msa: bool = True
    state: str = "full"

    @property
    def id(self):
        return self.name if self.state == "full" else f"{self.name}-{self.state}"

    @property
    def arch(self):
        return synth.MsaArch(self.layers, self.d, self.heads, 2 * self.d, embed_positions_msa=self.embed_positions_msa,
                             msa_pos_dim=self.msa_pos_dim, max_positions=1024)

    @property
    def seed(self):
        return 1000 + sum(map(ord, self.name))

    def cols(self):
        if self.positions:
            return list(self.positions)
        return sorted({0, 1, self.C // 2, self.C - 1} & set(range(self.C)))

    def raw_state(self):
        st = synth.make_msa_state(self.arch, self.seed, qk_gain=1.0)
        blk = {"row-only": "column_self_attention", "column-only": "row_self_attention"}.get(self.state)
        if blk:
            for i in range(self.layers):
                for t in ("weight", "bias"):
                    st[f"layers.{i}.{blk}.layer.out_proj.{t}"].zero_()
        return st

    def tokens(self):
        """int32 [R, C]: a random alignment of a random protein of C - 1 residues, BOS column first."""
        rows = synth.random_alignment(synth.random_protein(self.C - 1, self.seed), self.R, self.seed + 1)
        return msa_engine.tokenize_alignment(rows)

    def reference(self, fault=None):
        """fp64 [len(cols), vocab] log-probs of the oracle (``fault``: one of msa_oracle.FAULTS)."""
        return MO.masked_marginal_table(self.raw_state(), torch.from_numpy(self.tokens()).long(), self.layers, self.heads,
                                        positions=self.cols(), dtype=torch.float64, fault=fault).numpy()

    def scorer(self, precision):
        arch = self.arch
        cfg = checkpoint.config_from_msa_synth(arch)
        st = checkpoint.normalise_msa_synth_state(arch, self.raw_state())
        Cw = min(self.C, 1024)
        max_rows = self.per_pass * self.R * Cw if self.per_pass else msa_engine.default_max_rows(cfg, self.R, Cw, want=4)
        return msa_engine.MsaScorer(cfg, st, precision=precision, max_rows=max_rows)


def _grid():
    out = []
    # Cw around the Kp (64) and Cp (128) padding: Cp 128 and 384 run the tied GEMMs single-CTA, Cp 256 as CTA pairs
    for C in (2, 64, 65, 128, 129, 257):
        out += [Case(f"cw{C}", C=C, state=s) for s in STATES]
    # R = 1: the column shortcut; 21 and 130: the score GEMM's K = 64 R spans two and seven hi*hi chunks, long row walks
    for R in (1, 2, 21, 130):
        out += [Case(f"r{R}", R=R, state=s) for s in STATES]
    # head counts whose gather / scatter / tied_col blocks are not whole warps
    out += [Case(f"h{H}", layers=1, d=64 * H, heads=H, R=3, C=33) for H in (1, 5, 12)]
    # alignments per pass (13 positions: 13 passes of 1, 3+3+3+3+1, 7+6)
    pos13 = (0, 1, 3, 7, 12, 16, 20, 25, 29, 33, 37, 39, 40)
    out += [Case(f"pass{n}", R=4, positions=pos13, per_pass=n) for n in (1, 3, 7)]
    # row positions: a full-width table, the first release's 1-wide one, none
    out += [Case("rowpos_d", R=6), Case("rowpos_1", R=6, msa_pos_dim=1), Case("rowpos_none", R=6, embed_positions_msa=False)]
    # 1100 columns: 1024-wide windows (1023 at the right edge), window start != 0 from position 513 on
    out += [Case("window", layers=1, d=64, heads=1, R=2, C=1100, positions=(0, 1, 511, 512, 550, 588, 589, 1099))]
    # one layer: the pruned last layer alone (the other cases have two)
    out += [Case("layers1", layers=1, C=65, state=s) for s in ("full", "row-only")]
    return out


CASES = _grid()


def max_err(got, ref):
    return float(np.abs(np.asarray(got, dtype=np.float64) - ref).max())
