"""CPU: ESM C (evoscale) host logic against the unmodified reference's goldens (oracle/gen_golden_esmc.py): the fp32 oracle reproduces
the reference's masked rows and score column, the window rule, mutant parsing and NaN semantics, the checkpoint loader's checks, the
fc1 gate/up interleave, and the drop-in CLI's flags."""
import json
import os
import re

import numpy as np
import pandas as pd
import pytest
import torch

from oracle import esmc_oracle as O
from proteingym_b200 import checkpoint, synth
from proteingym_b200.mutants import parse_esmc_mutants
from proteingym_b200.windows import esmc_window_rows, esmc_window_starts

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ESMC_GOLDENS = ["esmc_300m", "esmc_600m", "esmc_300m_window"]


def load_esmc_golden(name):
    """-> dict(meta, arch, seq, df (reference CLI output), table (reference masked rows in scoring order), positions (0-based residues,
    sorted), state() (the seeded weights, regenerated))."""
    with open(os.path.join(GOLDEN, f"{name}_meta.json")) as fh:
        meta = json.load(fh)
    a = meta["arch"]
    arch = synth.EsmcArch(a["layers"], a["embed_dim"], a["ffn_dim"])
    df = pd.read_csv(os.path.join(GOLDEN, f"{name}_reference_output.csv"))
    seq = meta["sequence"]
    pos = sorted({p for m in df["mutant"] for p, _, _ in (O.parse(str(m), seq) or [])})
    return dict(meta=meta, arch=arch, seq=seq, df=df, table=np.load(os.path.join(GOLDEN, f"{name}_reference_table.npy")), positions=pos,
                state=lambda: synth.make_esmc_state(arch, seed=meta["seed"]))


@pytest.mark.parametrize("name", ESMC_GOLDENS)
def test_oracle_reproduces_reference_golden(name):
    g = load_esmc_golden(name)
    assert g["table"].shape == (len(g["positions"]), 64)
    st = g["state"]()
    pos = g["positions"]
    rows = O.masked_rows(st, g["seq"], pos, torch.float32)
    assert np.abs(rows.numpy() - g["table"]).max() <= 1e-5
    want = g["df"][g["meta"]["score_column"]].to_numpy()
    got = O.score_mutants(g["df"]["mutant"], g["seq"], {p: rows[i] for i, p in enumerate(pos)})
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.isnan(want).sum() >= 5
    assert np.nanmax(np.abs(got - want)) <= 1e-5


@pytest.mark.parametrize("L", [1022, 1023, 1100, 3423])
def test_window_starts_follow_reference_rule(L):
    edges = [0, 1, 2, 3, 509, 510, 511, 512, 513, 514, L // 2, L - 513, L - 512, L - 511, L - 510, L - 509, L - 3, L - 2, L - 1]
    edges = [p for p in edges if 0 <= p < L]
    starts, T = esmc_window_starts(edges, L)
    assert T == min(L + 2, 1024)
    for p, s in zip(edges, starts):
        assert (s, min(L, s + 1022)) == O.window(p, L)
        assert s <= p < s + T - 2
    res = np.arange(L, dtype=np.int32) % 20 + 4
    tok, positions, win_start, T = esmc_window_rows(res, edges, 0, 2)
    for p, q, w in zip(edges, positions, win_start):
        s, e = O.window(p, L)
        assert list(tok[w:w + T]) == [0] + list(res[s:e]) + [2] and tok[q] == res[p] and q - w == p - s + 1


def test_mutant_parsing_and_nan_semantics():
    seq = "MKVLAG"
    muts = ["M1A", "K2R:V3L", "M1AXYZ", "m1A", "A1M", "M0A", "M7A", "K2R:bad", "K2R:", "12", "M01C", "K2R:K2C"]
    pos, wt, mt, offs, valid = parse_esmc_mutants(muts, seq)
    want_valid = [O.parse(m, seq) is not None for m in muts]
    assert valid.tolist() == want_valid == [True, True, True, False, False, False, False, False, False, False, True, True]
    assert offs.tolist() == [0, 1, 3, 4, 4, 4, 4, 4, 4, 4, 4, 5, 7] and pos.tolist() == [0, 1, 2, 0, 0, 1, 1]
    with pytest.raises(KeyError):  # a mutant letter outside the 20 amino acids: the reference's aa_to_token lookup raises
        parse_esmc_mutants(["M1B"], seq)
    rows = {p: torch.arange(64, dtype=torch.float64) * (p + 1) for p in range(len(seq))}
    s = O.score_mutants(muts, seq, rows)
    assert np.isnan(s).tolist() == [not v for v in want_valid]


def test_loader_checks_keys_shapes_and_release_dims(tmp_path):
    arch = synth.EsmcArch(2, 128, 256)
    st = synth.make_esmc_state(arch, seed=4)
    conf = checkpoint.esmc_config_from_state(st)
    assert (conf.arch, conf.layers, conf.embed_dim, conf.heads, conf.ffn_dim, conf.vocab) == ("esmc", 2, 128, 2, 256, 64)
    bad = dict(st)
    del bad["transformer.blocks.1.attn.k_ln.weight"]
    with pytest.raises(ValueError, match="k_ln"):
        checkpoint.esmc_config_from_state(bad)
    bad = dict(st)
    bad["transformer.blocks.0.ffn.3.weight"] = torch.zeros(128, 255)
    with pytest.raises(ValueError, match="ffn.3"):
        checkpoint.esmc_config_from_state(bad)
    snap = tmp_path / "snap"
    f = synth.write_esmc_checkpoint(str(snap / "data/weights/esmc_300m_2024_12_v0.pth"), arch, state={k: v.half() for k, v in st.items()})
    with pytest.raises(ValueError, match="not esmc_300M"):
        checkpoint.load_esmc_checkpoint("esmc_300M", str(snap))
    assert checkpoint.resolve_esmc_weights("esmc_300M", str(snap)) == str(snap / "data/weights/esmc_300m_2024_12_v0.pth")
    assert checkpoint.resolve_esmc_weights("esmc_300M", str(snap / "data/weights/esmc_300m_2024_12_v0.pth")).endswith(".pth")
    with pytest.raises(FileNotFoundError, match="never downloaded"):
        os.environ["HF_HUB_CACHE"] = str(tmp_path / "empty_cache")
        try:
            checkpoint.resolve_esmc_weights("esmc_600M")
        finally:
            del os.environ["HF_HUB_CACHE"]
    assert f is not None
    cos, sin = checkpoint.esmc_rotary_tables(1024)
    ocos, osin = O.rotary_tables(1024, torch.float32)
    assert torch.equal(cos, ocos) and torch.equal(sin, osin)


def test_fc1_interleave_is_a_permutation():
    """The row order pg_load_weights gives fc1 (api.cu interleave_gate_up_kernel), restated: rows 16i..16i+7 = gate rows 8i..8i+7,
    rows 16i+8..16i+15 = up rows 8i..8i+7."""
    src = pathlib_src()
    assert "const int sr = c < 8 ? 8 * blk + c : f + 8 * blk + (c - 8);" in src
    for f in (256, 2560, 3072):
        r = np.arange(2 * f)
        blk, c = r // 16, r % 16
        sr = np.where(c < 8, 8 * blk + c, f + 8 * blk + c - 8)
        assert np.array_equal(np.sort(sr), r)
        assert np.all(sr[(c < 8)] < f) and np.all(sr[(c >= 8)] >= f)
        assert np.array_equal(sr[c < 8] + f, sr[c >= 8])  # gate column j and up column j land in one fragment (blocks 2i, 2i + 1)


def pathlib_src():
    with open(os.path.join(os.path.dirname(GOLDEN), "..", "proteingym_b200", "csrc", "api.cu")) as fh:
        return fh.read()


def test_cli_flags_match_reference():
    from proteingym_b200 import score_evoscale
    with open(os.path.join(GOLDEN, "esmc_cli_flags.json")) as fh:
        ref = json.load(fh)
    acts = {a.option_strings[0]: a for a in score_evoscale.create_parser()._actions if a.dest != "help"}
    for flag, r in ref.items():
        a = acts[flag]
        assert (a.dest, a.default, a.required) == (r["dest"], r["default"], r["required"]), flag
        assert (list(a.choices) if a.choices else None) == r["choices"] and (a.nargs == 0) == r["store_true"], flag
    assert set(acts) - set(ref) == {"--precision", "--device"}
    assert re.search(r"NotImplementedError", open(score_evoscale.__file__).read())
