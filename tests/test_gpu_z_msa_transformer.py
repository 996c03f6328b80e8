"""GPU (-m gpu): the MSA Transformer path (tied row attention as grouped wgmma GEMMs, column attention through the wgmma attention
kernel, pg_msa_masked_marginals) against golden vectors of the unmodified reference and the CPU oracle. Tolerance: 1e-3 abs per mutant
score in the parity modes (north_star's bar); f16 is held to the bound of tests/test_gpu_z_msa_fp64.py."""
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest
import torch

from conftest import ROOT
from msa_fp64_cases import BOUND
from msa_transformer_cases import case_dir, have, load_case
from oracle import msa_oracle as MO
from proteingym_b200 import _lib, checkpoint, msa_engine, synth

pytestmark = pytest.mark.gpu
TOL = 1e-3
MODES = ["f16f8", "f16x3"]


def make_scorer(arch, seed, precision, R, C, qk_gain=2.0):
    cfg = checkpoint.config_from_msa_synth(arch)
    st = checkpoint.normalise_msa_synth_state(arch, synth.make_msa_state(arch, seed, qk_gain=qk_gain))
    return msa_engine.MsaScorer(cfg, st, precision=precision, max_rows=msa_engine.default_max_rows(cfg, R, min(C, 1024), want=3))


@pytest.mark.parametrize("precision", MODES + ["f16"])
@pytest.mark.parametrize("name", ["tiny", "weights", "batched"])
def test_golden_table_and_scores(name, precision):
    c = load_case(name)
    arch, meta = c["arch"], c["meta"]
    toks = msa_engine.tokenize_alignment(c["rows"])
    sc = make_scorer(arch, meta["seed"], precision, *toks.shape)
    tab = sc.masked_marginal_rows(toks, meta["table_positions"]).cpu().numpy()
    col = f"{meta['column']}_seed{meta['seeds'][0]}"
    got = sc.score_assay(c["rows"], c["sequence"], list(c["df"]["mutant"]), meta["MSA_start"])
    sc.close()
    et, es = np.abs(tab - c["table"]).max(), np.abs(got - c["df"][col].to_numpy()).max()
    print(f"\nMSA Transformer {name} {precision}: max|dlogp|={et:.2e} max|dscore|={es:.2e}")
    if precision == "f16":  # a score is a difference of two log-probs
        assert et < BOUND["f16"] and es < 2 * BOUND["f16"]
    else:
        assert et < TOL and es < TOL


@pytest.mark.parametrize("precision", MODES)
def test_golden_windows(precision):
    """1101 columns: per-position 1024-column windows (1023 at the right edge) as the reference slices them."""
    c = load_case("window")
    arch, meta = c["arch"], c["meta"]
    toks = msa_engine.tokenize_alignment(c["rows"])
    sc = make_scorer(arch, meta["seed"], precision, toks.shape[0], 1024)
    tab = sc.masked_marginal_rows(toks, meta["table_positions"]).cpu().numpy()
    col = f"{meta['column']}_seed{meta['seeds'][0]}"
    got = sc.score_assay(c["rows"], c["sequence"], list(c["df"]["mutant"]), meta["MSA_start"])
    sc.close()
    assert np.abs(tab - c["table"]).max() < TOL and np.abs(got - c["df"][col].to_numpy()).max() < TOL


@pytest.mark.parametrize("precision", MODES)
def test_golden_true_size_msa1b(precision):
    """12 x 768, 12 heads, ffn 3072 (MSA-1b): 48 sampled rows x 130 columns, reference CLI output + 18 rows of its table."""
    if not have("msa1b"):
        pytest.skip("true-size fixture not generated")
    c = load_case("msa1b")
    arch, meta = c["arch"], c["meta"]
    toks = msa_engine.tokenize_alignment(c["rows"])
    sc = make_scorer(arch, meta["seed"], precision, *toks.shape, qk_gain=c["qk_gain"])
    tab = sc.masked_marginal_rows(toks, meta["table_positions"]).cpu().numpy()
    col = f"{meta['column']}_seed{meta['seeds'][0]}"
    got = sc.score_assay(c["rows"], c["sequence"], list(c["df"]["mutant"]), meta["MSA_start"])
    sc.close()
    ref = c["df"][col].to_numpy()
    nsites = c["df"]["mutant"].str.count(":").to_numpy() + 1
    err = np.abs(got - ref)
    print(f"\nMSA-1b true size {precision}: max|dlogp|={np.abs(tab - c['table']).max():.2e} max|dscore|={err.max():.2e} "
          f"(1 site {err[nsites == 1].max():.2e}) mean={err.mean():.2e}")
    assert np.abs(tab - c["table"]).max() < TOL and err.max() < TOL


def test_results_do_not_depend_on_the_pass_split_and_single_row_alignment():
    """Positions processed one per pass or several per pass give the same bits; an alignment of ONE row takes the reference's
    column-attention shortcut (v -> out_proj, axial_attention.py:266-278), which the general kernel reproduces."""
    arch = synth.MsaArch(2, 128, 2, 256)
    t = synth.random_protein(70, seed=3)
    rows = synth.random_alignment(t, 9, seed=4)
    toks = msa_engine.tokenize_alignment(rows)
    cfg = checkpoint.config_from_msa_synth(arch)
    st = checkpoint.normalise_msa_synth_state(arch, synth.make_msa_state(arch, 5))
    pos = list(range(0, 71, 5))
    a = msa_engine.MsaScorer(cfg, st, precision="f16f8", max_rows=toks.size)          # one alignment per pass
    b = msa_engine.MsaScorer(cfg, st, precision="f16f8", max_rows=7 * toks.size)      # seven per pass
    ta, tb = a.masked_marginal_rows(toks, pos), b.masked_marginal_rows(toks, pos)
    assert torch.equal(ta, tb)
    one = b.masked_marginal_rows(toks[:1], pos).cpu().numpy()
    a.close(); b.close()
    ref = MO.masked_marginal_table(synth.make_msa_state(arch, 5), torch.from_numpy(toks[:1]).long(), arch.layers, arch.heads, positions=pos)
    assert np.abs(one - ref.numpy()).max() < TOL


def test_bad_calls_fail_loudly():
    arch = synth.MsaArch(1, 64, 1, 128)
    cfg = checkpoint.config_from_msa_synth(arch)
    st = checkpoint.normalise_msa_synth_state(arch, synth.make_msa_state(arch, 1))
    sc = msa_engine.MsaScorer(cfg, st, precision="f16x3", max_rows=4096)
    toks = msa_engine.tokenize_alignment(synth.random_alignment(synth.random_protein(30, 1), 4, 2))
    with pytest.raises(IndexError):
        sc.masked_marginal_rows(toks, [31])
    with pytest.raises(_lib.PgError, match="exceeds the workspace"):
        sc.masked_marginal_rows(np.tile(toks, (40, 1)), [3])
    bad = toks.copy(); bad[2, 5] = 1
    with pytest.raises(ValueError, match="padding"):
        sc.masked_marginal_rows(bad, [3])
    with pytest.raises(RuntimeError, match="unaligned"):
        msa_engine.tokenize_alignment([("a", "MKV"), ("b", "MK")])
    # an ESM entry point on an MSA handle
    out = torch.empty((1, 33), device="cuda")
    tok = torch.zeros(8, dtype=torch.int32, device="cuda")
    assert sc.lib.pg_masked_marginals(sc.handle, tok.data_ptr(), 8, tok.data_ptr(), None, None, 1, 8, out.data_ptr(), None) != 0
    sc.close()


def test_cli_matches_reference_csv(tmp_path):
    """proteingym_b200/compute_fitness.py --model_type MSA_transformer on the files the reference CLI ran on: same columns (two seed
    columns + ensemble), scores within 1e-3; weights recomputed on the GPU equal the reference's numba weights."""
    c = load_case("weights")
    meta, arch = c["meta"], c["arch"]
    ck = str(tmp_path / "msa_synth.pt")
    synth.write_msa_checkpoint(ck, arch, seed=meta["seed"])
    os.makedirs(tmp_path / "msa"); os.makedirs(tmp_path / "dms"); os.makedirs(tmp_path / "w"); os.makedirs(tmp_path / "out")
    import shutil
    shutil.copy(os.path.join(c["dir"], "alignment.a2m"), tmp_path / "msa" / "weights.a2m")
    shutil.copy(os.path.join(c["dir"], "dms.csv"), tmp_path / "dms" / "weights.csv")
    pd.DataFrame({"DMS_id": ["OTHER", "weights"], "DMS_filename": ["other.csv", "weights.csv"], "target_seq": ["MKV", meta["target_seq"]],
                  "MSA_filename": ["other.a2m", "weights.a2m"], "MSA_start": [1, meta["MSA_start"]], "MSA_end": [3, meta["MSA_end"]],
                  "weight_file_name": ["other.npy", "weights.npy"]}).to_csv(tmp_path / "map.csv", index=False)
    cmd = [sys.executable, os.path.join(ROOT, "proteingym_b200", "compute_fitness.py"), "--model-location", ck, "--model_type", "MSA_transformer",
           "--dms_index", "1", "--dms_mapping", str(tmp_path / "map.csv"), "--dms-input", str(tmp_path / "dms"), "--dms-output", str(tmp_path / "out"),
           "--scoring-strategy", "masked-marginals", "--msa-path", str(tmp_path / "msa"), "--msa-weights-folder", str(tmp_path / "w"),
           "--msa-samples", str(meta["msa_samples"]), "--seeds", *[str(s) for s in meta["seeds"]]]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    got = pd.read_csv(tmp_path / "out" / "weights.csv")
    ref = c["df"]
    assert list(got.columns) == list(ref.columns)
    for col in ref.columns:
        if col.startswith("msa_synth"):
            assert np.abs(got[col].to_numpy() - ref[col].to_numpy()).max() < TOL, col
    w = np.load(tmp_path / "w" / "weights.npy")
    assert np.allclose(w, c["weights"], rtol=0, atol=1e-12)
    # second run: every seed column exists -> skipped, file unchanged (compute_fitness.py:365-372)
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "Skipping seed" in r.stdout


@pytest.mark.parametrize("G,rows_a,N,rows_b,K,nseg,epi", [(3, 128, 100, 100, 128, 3, 2), (4, 256, 304, 384, 192, 3, 0), (2, 384, 513, 640, 1024, 1, 2),
                                                          (5, 128, 64, 64, 64, 3, 0), (2, 640, 513, 640, 2560, 3, 2), (3, 256, 3200, 3200, 192, 3, 0)])
@pytest.mark.parametrize("cta2", [0, 1])
def test_grouped_gemm_matches_fp64(G, rows_a, N, rows_b, K, nseg, epi, cta2):
    """The block-diagonal form of the wgmma GEMM the tied row attention uses (scores: epi 2 into fp32; context: epi 0 into fp16
    hi/lo planes): group g multiplies rows [g*rows_a, (g+1)*rows_a) of a with rows [g*rows_b, g*rows_b + N) of w."""
    import ctypes as C
    lib = _lib.load()
    lib.pg_set_tuning(b"gemm_cta2", cta2)
    g = torch.Generator(device="cuda").manual_seed(G + rows_a + N + K)
    A = torch.randn(G * rows_a, K, device="cuda", generator=g)
    W = torch.randn(G * rows_b, K, device="cuda", generator=g) / K ** 0.5

    def hilo(t):
        hi = t.to(torch.float16)
        return torch.cat([hi, (t - hi.float()).to(torch.float16)], dim=1).contiguous()
    a16, w16 = (hilo(A), hilo(W)) if nseg == 3 else (A.half().contiguous(), W.half().contiguous())
    Ad = a16[:, :K].double() + (a16[:, K:].double() if nseg == 3 else 0)
    Wd = w16[:, :K].double() + (w16[:, K:].double() if nseg == 3 else 0)
    ref = torch.stack([Ad[i * rows_a:(i + 1) * rows_a] @ Wd[i * rows_b:i * rows_b + N].T for i in range(G)]).reshape(G * rows_a, N)
    if nseg == 3:  # the kernel drops lo*lo
        ref = ref - torch.stack([a16[i * rows_a:(i + 1) * rows_a, K:].double() @ w16[i * rows_b:i * rows_b + N, K:].double().T
                                 for i in range(G)]).reshape(G * rows_a, N)
    args = _lib.PgGemmArgs()
    args.a, args.lda, args.w, args.ldw = a16.data_ptr(), a16.shape[1], w16.data_ptr(), w16.shape[1]
    args.M, args.N, args.K, args.nseg, args.epi = G * rows_a, N, K, nseg, epi
    args.grp_rows_a, args.grp_rows_b = rows_a, rows_b
    npl = 2 if nseg == 3 else 1
    ldr = (N + 3) // 4 * 4
    if epi == 2:
        resid = torch.zeros(G * rows_a, ldr, device="cuda")
        args.resid, args.ldr = resid.data_ptr(), ldr
    else:
        out = torch.zeros(G * rows_a, N * npl, device="cuda", dtype=torch.float16)
        args.out_h, args.ldo, args.out_lo_off = out.data_ptr(), N * npl, (N if nseg == 3 else 0)
    try:
        _lib.check(lib.pg_gemm(C.byref(args), None))
        torch.cuda.synchronize()
    finally:
        lib.pg_set_tuning(b"gemm_cta2", 1)
    got = resid[:, :N].double() if epi == 2 else out[:, :N].double() + (out[:, N:].double() if nseg == 3 else 0)
    err, amax = (got - ref).abs().max().item(), ref.abs().max().item()
    bound = 4e-7 * (K * nseg) ** 0.5 * max(4.0, amax) if (epi == 2 or nseg == 3) else 2.5e-3 * max(1.0, amax / 4)
    assert err < bound, (err, bound)


def test_two_gpu_position_partition_is_bit_identical():
    """MsaScorer.score_assay(shard=(rank, world)) over NCCL on 2 GPUs: every rank ends with the single-GPU scores, bit for bit.
    Needs 2 devices (skipped on the 1-GPU box; runs under `gpurun --gpus 2`)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29673", os.path.join(ROOT, "scripts", "check_msa_partition.py")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "bit_identical=True" in r.stdout
