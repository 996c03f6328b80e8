"""PoET on the H100 against the goldens the unmodified reference wrote (tests/golden/poet_goldens.jsonl): every case through
score_poet.main, failures included; pass-size independence; the neighbour counts; refused configurations. Weights are regenerated from
the recorded seeds."""
import ctypes as C
import json
import os

import numpy as np
import pandas as pd
import pytest
import torch

from proteingym_b200 import _lib, checkpoint, synth
from proteingym_b200 import poet_engine as E
from proteingym_b200 import score_poet

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = [json.loads(ln) for ln in open(os.path.join(ROOT, "tests", "golden", "poet_goldens.jsonl"))]
BAR = 1e-3


def _write_inputs(case, tmp):
    for sub in ("dms", "msa", "out"):
        os.makedirs(os.path.join(tmp, sub), exist_ok=True)
    ref = case["ref"]
    pd.DataFrame({"mutated_sequence": case["variants"]}).to_csv(os.path.join(tmp, "dms", ref["DMS_filename"]), index=False)
    pd.DataFrame([dict(DMS_id=case["name"], **ref)]).to_csv(os.path.join(tmp, "ref.csv"), index=False)
    stem = os.path.splitext(ref["DMS_filename"])[0]
    with open(os.path.join(tmp, "msa", stem + ".a3m.zst"), "w") as fh:
        for i, r in enumerate(case["a3m"]):
            fh.write(f">seq{i}\n{r}\n")
    ckpt = os.path.join(tmp, "poet.ckpt")
    synth.write_poet_checkpoint(ckpt, synth.PoetArch(**case["arch"]), seed=case["seed"])
    return ckpt


def _run(case, tmp, precision):
    ckpt = _write_inputs(case, tmp)
    argv = ["--checkpoint", ckpt, "--DMS_reference_file_path", os.path.join(tmp, "ref.csv"), "--DMS_data_folder", os.path.join(tmp, "dms"),
            "--DMS_index", "0", "--output_scores_folder", os.path.join(tmp, "out"), "--MSA_folder", os.path.join(tmp, "msa"),
            "--precision", precision] + case["flags"]
    return score_poet.main(score_poet.create_parser().parse_args(argv))


@pytest.mark.parametrize("precision", ["auto", "f16x3", "f16f8", "f16"])
@pytest.mark.parametrize("case", CASES, ids=lambda c: c["name"])
def test_golden_case(case, precision, tmp_path):
    if "error" in case:  # the same failure at the same step as the reference
        wt = case["ref"]["target_seq"][case["ref"]["MSA_start"] - 1:case["ref"]["MSA_end"]]
        step = "all gaps" if "error" in case["sampler"] else ("not the wild type" if case["a3m"][0] != wt else "contains a gap")
        with pytest.raises(AssertionError, match=step):
            _run(case, str(tmp_path), precision)
        return
    out = _run(case, str(tmp_path), precision)
    assert list(out.columns) == case["out_columns"]
    got = out["PoET_score"].to_numpy(dtype=np.float64)
    ref = np.array([np.nan if v is None else v for v in case["scores"]], dtype=np.float64)
    assert (np.isnan(got) == np.isnan(ref)).all()
    err = float(np.nanmax(np.abs(got - ref)))
    print(f"POET_ERR {case['name']} {precision} {err:.3e}")
    if precision in ("auto", "f16x3", "f16f8"):
        assert err <= BAR, err
    else:  # single fp16: not a parity mode
        assert err <= 0.5, err


def test_pass_split_is_bit_identical(tmp_path):
    case = next(c for c in CASES if c["name"] == "long_context")
    ckpt = _write_inputs(case, str(tmp_path))
    conf, st = checkpoint.load_poet_checkpoint(ckpt)
    seqs = [r.encode() for r in case["a3m"]]
    ctx = E.sample_context(seqs, np.arange(len(seqs)), 150, 1)  # <= 244 rows: fits both workspaces
    variants = [E.append_startstop(E.encode(v.encode())) for v in case["variants"]] * 7
    res = []
    for max_rows in (8192, 250):  # one pass, and passes of 2 rows
        sc = E.PoetScorer(conf, st, 256, precision="f16x3", max_rows=max_rows)
        try:
            sc.set_context(ctx)
            res.append(sc.loglik(variants))
        finally:
            sc.close()
    assert np.array_equal(res[0], res[1])


def test_neighbor_counts_exact():
    for case in CASES:
        if "idxs" not in case["sampler"]:
            continue
        msa = E.weight_matrix([r.encode() for r in case["a3m"]])
        masked = np.where(msa == E.GAP, 255, msa)
        sim = (msa[:, None, :] == masked[None, :, :]).sum(axis=2) / (msa != E.GAP).sum(axis=1, keepdims=True)
        assert E.neighbor_counts(msa).tolist() == ((1 - sim) <= E.THETA).sum(axis=1).tolist()


def test_refused_configurations():
    lib = _lib.load()
    for heads, prec in ((4, _lib.PG_PREC_F16X3), (2, _lib.PG_PREC_F16D)):
        desc = _lib.PgModelDesc(arch=_lib.PG_ARCH_POET, layers=1, embed_dim=128, heads=heads, ffn_dim=512, vocab=24, max_positions=64,
                                precision=prec, device=0)
        h = C.c_void_p()
        assert lib.pg_create(C.byref(desc), C.byref(h)) == 4  # PG_ERR_UNSUPPORTED


# ---- per token against the fp64 oracle (oracle/poet_oracle.py) at true width, 2 layers -------------------------------------------
TOKEN_BOUND = {"f16x3": 5e-5, "f16f8": 2e-4, "f16": 2e-2}  # measured: 1.0e-5, 5.7e-5 (before the 64-element K chunks), 1.6e-3
VARIANT_T = [2, 63, 64, 65, 127, 128, 129, 1023]
CONTEXT_TM = [1, 63, 64, 65, 6145, 24640]
_ORACLES = {}


def _true_width():
    import sys
    sys.path.insert(0, ROOT)
    from oracle.poet_oracle import PoetOracle
    if not _ORACLES:
        arch = synth.PoetArch(2, 1024, 16)
        st = synth.make_poet_state(arch, seed=7)
        conf = checkpoint.PoetConfig(arch.layers, arch.hidden_dim, arch.heads, 4096, False)
        _ORACLES["st"] = (conf, st)
        _ORACLES["f64"] = PoetOracle(st, 2, 16, torch.float64, "cuda")
        _ORACLES["f32"] = PoetOracle(st, 2, 16, torch.float32, "cuda")
    return _ORACLES


def _segments(Tm, rng):
    """Unequal segments <start> residues <stop> summing to Tm."""
    lens = []
    while sum(lens) < Tm:
        lens.append(min(int(rng.integers(3, 700)), Tm - sum(lens)))
    rows = []
    for n in lens:
        r = rng.integers(0, 20, size=n).astype(np.int64)
        r[0] = E.START
        if n > 1:
            r[-1] = E.STOP
        rows.append(r)
    return rows


def _variants(rng):
    out = []
    for T in VARIANT_T:
        r = np.concatenate([[E.START], rng.integers(0, 20, size=T - 2), [E.STOP]])[:T].astype(np.int64)
        if T > 10:
            r[5] = E.MASK  # an X inside: its target is ignored
        out.append(r)
    return out


@pytest.mark.parametrize("precision", list(TOKEN_BOUND))
def test_token_logp_and_record_vs_fp64_oracle(precision):
    o = _true_width()
    conf, st = o["st"]
    rng = np.random.default_rng(3)
    variants = _variants(rng)
    sc = E.PoetScorer(conf, st, 1100, precision=precision)
    try:
        for Tm in CONTEXT_TM:
            ctx = _segments(Tm, rng)
            sc.set_context(ctx)
            ids = torch.from_numpy(np.concatenate(ctx))
            rec = o["f64"].context(ids, [len(r) for r in ctx])
            for layer in range(conf.layers):  # the record: rotated keys and values, per layer
                k, v = sc.record(layer)
                kr, vr = rec[layer][0].flatten(1), rec[layer][1].flatten(1)
                ek = float((k.double() - kr).abs().max() / kr.abs().max())
                ev = float((v.double() - vr).abs().max() / vr.abs().max())
                assert ek <= (5e-3 if precision == "f16" else 2e-5) and ev <= (5e-3 if precision == "f16" else 2e-5), (Tm, layer, ek, ev)
            _, tok = sc.loglik(variants, tok_logp=True)
            rec32 = o["f32"].context(ids, [len(r) for r in ctx]) if precision == "f16x3" else None
            worst, worst32 = 0.0, 0.0
            for i, r in enumerate(variants):
                ref = o["f64"].token_logp(torch.from_numpy(r), rec).cpu().numpy()
                err = np.abs(tok[i, :len(r) - 1] - ref)
                assert (tok[i, len(r) - 1:] == 0).all()
                worst = max(worst, float(err.max()))
                if rec32 is not None:
                    r32 = o["f32"].token_logp(torch.from_numpy(r), rec32).double().cpu().numpy()
                    worst32 = max(worst32, float(np.abs(r32 - ref).max()))
            print(f"POET_TOKEN {precision} Tm={Tm} max|dlogp|={worst:.3e}" + (f" torch-fp32={worst32:.3e}" if rec32 is not None else ""))
            assert worst <= TOKEN_BOUND[precision], (Tm, worst)
    finally:
        sc.close()


def test_true_shape_golden_per_token_evidence(tmp_path):
    """Where the 12 x 1024 golden's score difference comes from: per-token |dlog p| of f16x3 and of torch fp32 against fp64 on its
    first member, same context, same variants."""
    import sys
    sys.path.insert(0, ROOT)
    from oracle.poet_oracle import PoetOracle
    case = next(c for c in CASES if c["name"] == "poet_true_shape")
    arch = synth.PoetArch(**case["arch"])
    st = synth.make_poet_state(arch, seed=case["seed"])
    conf = checkpoint.PoetConfig(arch.layers, arch.hidden_dim, arch.heads, arch.ff_dim or 4 * arch.hidden_dim, arch.norm)
    seqs = [r.encode() for r in case["a3m"]]
    msa = E.weight_matrix(seqs)
    f = case["flags"]
    seed = int(f[f.index("--seed") + 1])
    ctx = E.sample_context(seqs, E.sample_idxs(msa, E.neighbor_counts(msa), 1.0, seed), int(f[1]), seed)
    variants = [E.append_startstop(E.encode(v.encode())) for v in case["variants"]]
    ids = torch.from_numpy(np.concatenate(ctx)).long()
    variants = [v.astype(np.int64) for v in variants]
    o64, o32 = PoetOracle(st, arch.layers, arch.heads, torch.float64, "cuda"), PoetOracle(st, arch.layers, arch.heads, torch.float32, "cuda")
    rec64, rec32 = o64.context(ids, [len(r) for r in ctx]), o32.context(ids, [len(r) for r in ctx])
    sc = E.PoetScorer(conf, st, 400, precision="f16x3")
    try:
        sc.set_context(ctx)
        _, tok = sc.loglik(variants, tok_logp=True)
    finally:
        sc.close()
    e_ours, e_32, s_ours, s_32 = [], [], [], []
    for i, r in enumerate(variants):
        ref = o64.token_logp(torch.from_numpy(r), rec64).cpu().numpy()
        r32 = o32.token_logp(torch.from_numpy(r), rec32).double().cpu().numpy()
        e_ours.append(np.abs(tok[i, :len(r) - 1] - ref).max())
        e_32.append(np.abs(r32 - ref).max())
        s_ours.append(abs(tok[i, :len(r) - 1].astype(np.float64).sum() - ref.sum()))
        s_32.append(abs(r32.sum() - ref.sum()))
    print(f"POET_TRUE_SHAPE per-token max f16x3={max(e_ours):.3e} torch-fp32={max(e_32):.3e}; "
          f"row-sum max f16x3={max(s_ours):.3e} torch-fp32={max(s_32):.3e}")
    assert max(e_ours) <= TOKEN_BOUND["f16x3"]
