"""GPU (-m gpu): ESM C (evoscale) masked marginals against the fp64 oracle at both releases' widths, the SwiGLU GEMM epilogue against
fp64, the refused configurations, the re-tokenised windows and NaN rows of the assay path, and the drop-in CLI end to end."""
import math

import numpy as np
import pandas as pd
import pytest
import torch

from oracle import esmc_oracle as O
from proteingym_b200 import _lib, checkpoint, synth

pytestmark = pytest.mark.gpu
TOL = 1e-3
# Two-layer models at each release's width / heads / SwiGLU width: s = sqrt(2/36) makes a missed or doubled residual scale obvious.
# Bounds on max |log-prob - fp64| over T in {2, 63, 64, 65, 129, 1024}: ~4x the worst measured on an H100 80GB HBM3 (worst of both
# widths: f16x3 2.5e-5, f16f8 1.2e-4, f16 3.5e-3).
FP64_ARCHS = {"300m": synth.EsmcArch(2, 960, 2560), "600m": synth.EsmcArch(2, 1152, 3072)}
FP64_BOUND = {"f16x3": 1e-4, "f16f8": 5e-4, "f16": 1.4e-2}


def scorer(state, precision="f16x3", max_rows=32768):
    from proteingym_b200.esm_engine import EsmScorer
    return EsmScorer(checkpoint.esmc_config_from_state(state), state, precision=precision, max_rows=max_rows)


@pytest.fixture(scope="module")
def fp64_models():
    out = {}
    for name, arch in FP64_ARCHS.items():
        st = synth.make_esmc_state(arch, seed=23)
        out[name] = (st, {k: v.double() for k, v in st.items()})
    return out


@pytest.mark.parametrize("mode", list(FP64_BOUND))
@pytest.mark.parametrize("name", list(FP64_ARCHS))
def test_masked_rows_match_fp64_oracle(name, mode, fp64_models):
    st, ost = fp64_models[name]
    sc = scorer(st, precision=mode, max_rows=65536)
    worst = {}
    for T in (2, 63, 64, 65, 129, 1024):
        seq = synth.random_protein(T - 2, T)
        pos = sorted({0, 1, T // 2, T - 2, T - 1})  # token indices, BOS and EOS included
        toks = O.tokenize(seq)
        tb = toks.unsqueeze(0).repeat(len(pos), 1)
        for r, i in enumerate(pos):
            tb[r, i] = O.MASK_IDX
        lp = torch.log_softmax(O.esmc_forward(ost, tb, torch.float64), -1)
        ref = torch.stack([lp[r, i] for r, i in enumerate(pos)]).numpy()
        got = sc.masked_marginal_rows(toks.to(torch.int32).cuda(), pos).cpu().numpy()
        worst[T] = float(np.abs(got - ref).max())
    sc.close()
    print(f"\nesmc {name} {mode}: max|dlogp| vs fp64 by T: " + ", ".join(f"{T}: {v:.2e}" for T, v in worst.items()))
    assert max(worst.values()) < FP64_BOUND[mode], worst


def test_forward_logprobs_full_table_matches_fp64(fp64_models):
    """pg_forward_logprobs runs the unpruned last layer (SwiGLU on every row) and the head on every row."""
    st, ost = fp64_models["300m"]
    sc = scorer(st, precision="f16x3")
    seq = synth.random_protein(150, 11)
    got = sc.wt_marginal_table(seq).cpu().double()
    sc.close()
    ref = torch.log_softmax(O.esmc_forward(ost, O.tokenize(seq)[None], torch.float64), -1)[0]
    err = (got - ref).abs().max().item()
    print(f"\nesmc full table f16x3: max|dlogp| = {err:.2e}")
    assert err < FP64_BOUND["f16x3"]


def test_assay_windows_and_nan_rows_match_oracle(fp64_models):
    """L = 1100 > 1022: windows re-tokenised as <cls> slice <eos> at the left edge, around 511, in the middle and at the right edge;
    unparsable, out-of-range and wild-type-mismatched mutants come back NaN where the reference writes NaN."""
    st, ost = fp64_models["300m"]
    L = 1100
    seq = synth.random_protein(L, 41)
    sites = [0, 1, 2, 3, 509, 510, 511, 512, 513, 514, 550, L - 513, L - 511, L - 509, L - 3, L - 2, L - 1]
    aa = "ACDEFGHIKLMNPQRSTVWY"
    sub = lambda p: f"{seq[p]}{p + 1}{aa[(aa.index(seq[p]) + 3) % 20]}"
    muts = [sub(p) for p in sites] + [f"{sub(3)}:{sub(550)}", "Z5A", f"{seq[0]}0A", f"{seq[0]}{L + 1}A", "garbage", f"{sub(10)}:junk"]
    sc = scorer(st, precision="f16x3")
    got = sc.score_assay(seq, muts)
    sc.close()
    want = O.score_assay(ost, seq, muts, torch.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.isnan(want).sum() == 5
    ok = ~np.isnan(want)
    err = np.abs(got[ok] - want[ok]).max()
    print(f"\nesmc windowed L={L}: max|dscore| = {err:.2e}")
    assert err < TOL


@pytest.mark.parametrize("out_fmt", [0, 1, 2])
def test_swiglu_gemm_epilogue_matches_fp64(out_fmt):
    """pg_gemm epi 5 on interleaved gate/up rows (fp16 hi/lo x3 operands), M not a multiple of 128, against fp64."""
    lib = _lib.load()
    M, K, f = 300, 256, 384
    g = torch.Generator().manual_seed(3)
    a32 = torch.randn(M, K, generator=g)
    w32 = torch.randn(2 * f, K, generator=g) / math.sqrt(K)
    blk = torch.arange(2 * f) // 16
    c = torch.arange(2 * f) % 16
    src = torch.where(c < 8, 8 * blk + c, f + 8 * blk + c - 8)
    wi = w32[src].contiguous()  # rows interleaved in blocks of 8, as pg_load_weights packs them
    dev = torch.device("cuda")
    a_d, w_d = a32.to(dev), wi.to(dev)
    ap = torch.empty(M, 2 * K, dtype=torch.float16, device=dev)
    wp = torch.empty(2 * f, 2 * K, dtype=torch.float16, device=dev)
    s = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.pg_pack_weight(a_d.data_ptr(), M, K, 1, ap.data_ptr(), None, s))
    _lib.check(lib.pg_pack_weight(w_d.data_ptr(), 2 * f, K, 1, wp.data_ptr(), None, s))
    ldo = 2 * f if out_fmt else f  # fp16 elements: f hi + (f lo | 2f bytes of e4m3 planes)
    out = torch.zeros(M, ldo, dtype=torch.float16, device=dev)
    args = _lib.PgGemmArgs(a=ap.data_ptr(), lda=2 * K, w=wp.data_ptr(), ldw=2 * K, bias=None, M=M, N=2 * f, K=K, nseg=3, epi=5,
                           out_h=out.data_ptr(), ldo=ldo, out_lo_off=f if out_fmt else 0, out_fmt=out_fmt, out_scale=2.0)
    _lib.check(lib.pg_gemm(C_ref(args), s))
    torch.cuda.synchronize()
    u = a32.double() @ w32.double().T
    want = (torch.nn.functional.silu(u[:, :f]) * u[:, f:]).numpy()
    o = out.cpu()
    hi = o[:, :f].double().numpy()
    if out_fmt == 1:
        got, bound = hi + o[:, f:].double().numpy(), 2e-5
    elif out_fmt == 2:  # the e4m3 lo8 plane carries lo * 2^11 * 2
        lo8 = o[:, f:].contiguous().view(torch.uint8)[:, :f].view(torch.float8_e4m3fn).double().numpy()
        got, bound = hi + lo8 / (2048 * 2.0), 2e-4
    else:
        got, bound = hi, 4e-3 * max(1.0, float(np.abs(want).max()))
    err = float(np.abs(got - want).max())
    print(f"\nepi 5 out_fmt {out_fmt}: max|err| = {err:.2e} (|y| max {np.abs(want).max():.2f})")
    assert err < bound


def C_ref(args):
    import ctypes
    return ctypes.byref(args)


def test_refused_configurations():
    st = synth.make_esmc_state(synth.EsmcArch(1, 128, 256), seed=1)
    with pytest.raises(_lib.PgError, match="F16D"):
        scorer(st, precision="f16d")
    conf = checkpoint.esmc_config_from_state(st)
    conf.heads = 4  # head_dim 32
    from proteingym_b200.esm_engine import EsmScorer
    with pytest.raises(_lib.PgError, match="head_dim"):
        EsmScorer(conf, st)


def test_cli_end_to_end_matches_oracle(tmp_path, fp64_models):
    """score_evoscale on a 2-layer model: the reference's columns and row order, scores within 1e-3 of the oracle, NaN rows, the
    appended summary, and an assay whose scoring fails (mutant letter outside the 20 amino acids) -> NaN correlation and no CSV."""
    from proteingym_b200 import score_evoscale
    st, ost = fp64_models["300m"]
    wdir = tmp_path / "snap"
    synth.write_esmc_checkpoint(str(wdir / "data/weights/esmc_300m_2024_12_v0.pth"), synth.EsmcArch(2, 960, 2560), state=st)
    seq = synth.random_protein(120, 5)
    muts = synth.sample_mutants(seq, 80, 2, multi_frac=0.2, max_sites=2) + ["Q0A", f"{seq[4]}5{seq[4]}:bad"]
    (tmp_path / "dms").mkdir()
    df = pd.DataFrame({"mutant": muts, "DMS_score": np.random.RandomState(0).randn(len(muts)), "extra": range(len(muts))})
    df.to_csv(tmp_path / "dms" / "A.csv", index=False)
    pd.DataFrame({"mutant": [f"{seq[0]}1J"], "DMS_score": [0.0]}).to_csv(tmp_path / "dms" / "B.csv", index=False)
    pd.DataFrame({"DMS_id": ["A", "B"], "target_seq": [seq, seq]}).to_csv(tmp_path / "ref.csv", index=False)
    argv = ["--model_type", "esmc_300M", "--model_path", str(wdir), "--reference_csv", str(tmp_path / "ref.csv"), "--dms_dir",
            str(tmp_path / "dms"), "--output_dir", str(tmp_path / "out"), "--precision", "f16x3"]
    # the loader checks the dims against the release table; the test widens that entry to its 2-layer model for the CLI run
    with pytest.raises(ValueError, match="not esmc_300M"):
        checkpoint.load_esmc_checkpoint("esmc_300M", str(wdir))
    orig = checkpoint.ESMC_RELEASES["esmc_300M"]
    checkpoint.ESMC_RELEASES["esmc_300M"] = (2, 960, 2560, orig[3])
    try:
        res = score_evoscale.main(score_evoscale.create_parser().parse_args(argv))
        score_evoscale.main(score_evoscale.create_parser().parse_args(argv + ["--DMS_index", "0"]))
    finally:
        checkpoint.ESMC_RELEASES["esmc_300M"] = orig
    got = pd.read_csv(tmp_path / "out" / "A.csv")
    assert list(got.columns) == ["mutant", "DMS_score", "extra", "esmc_300M_score"] and got["mutant"].tolist() == muts
    want = O.score_assay(ost, seq, muts, torch.float64)
    g = got["esmc_300M_score"].to_numpy()
    assert np.array_equal(np.isnan(g), np.isnan(want)) and np.isnan(want).sum() == 2
    assert np.nanmax(np.abs(g - want)) < TOL
    assert not (tmp_path / "out" / "B.csv").exists() and math.isnan(res["B"]) and not math.isnan(res["A"])
    summ = pd.read_csv(tmp_path / "out" / "correlation_summary_esmc_300M.csv")
    assert summ["assay"].tolist() == ["A", "B", "A"]
    with pytest.raises(NotImplementedError):
        score_evoscale.main(score_evoscale.create_parser().parse_args(argv[:0] + ["--model_type", "esm3_open"] + argv[2:]))


@pytest.mark.parametrize("mode", ["f16x3", "f16f8", "auto"])
@pytest.mark.parametrize("name", ["esmc_300m", "esmc_600m", "esmc_300m_window"])
def test_golden_true_size_matches_reference(name, mode):
    """The unmodified reference's CLI output at true size (oracle/gen_golden_esmc.py): per-mutant scores within 1e-3, its masked rows
    within 2e-4 (f16x3) / 5e-4 (f16f8), NaN rows where it has them; `auto` stays within the bound of the scheme it picks."""
    from test_esmc_cpu import load_esmc_golden
    from proteingym_b200.esm_engine import choose_precision
    g = load_esmc_golden(name)
    st = g["state"]()
    prec = choose_precision(checkpoint.esmc_config_from_state(st), list(g["df"]["mutant"])) if mode == "auto" else mode
    sc = scorer(st, precision=prec, max_rows=65536)
    got = sc.score_assay(g["seq"], list(g["df"]["mutant"]))
    rows = sc.esmc_rows(g["seq"], g["positions"]).cpu().numpy()
    sc.close()
    want = g["df"][g["meta"]["score_column"]].to_numpy()
    assert np.array_equal(np.isnan(got), np.isnan(want))
    err, terr = float(np.nanmax(np.abs(got - want))), float(np.abs(rows - g["table"]).max())
    print(f"\n{name} {mode} ({prec}): max|dscore|={err:.2e} max|dlogp|={terr:.2e}")
    assert err < TOL and terr < (5e-4 if prec == "f16f8" else 2e-4)
