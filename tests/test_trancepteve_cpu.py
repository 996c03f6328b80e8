"""Host logic of the TranceptEVE / retrieval rows (SURVEY.md §8 a19, a21, a22) against outputs of the reference's UNMODIFIED
TrancepteveLMHeadModel (tests/golden/trancepteve_*, written by oracle/gen_golden_trancepteve.py). No GPU: the device half is
replaced by the oracle's CPU forward (tests/cpu_trancepteve.py); what is under test is proteingym_b200's alignment processing,
EVE-prior sampling, depth ladder, recalibration, window / prior-row arithmetic and score assembly."""
import json
import os
import pickle

import numpy as np
import pandas as pd
import pytest
import torch

from conftest import GOLDEN
from trancepteve_cases import SMALL_CASES as CASES, make_inputs

from proteingym_b200 import eve_prior, synth
from proteingym_b200.msa_processing import MSAProcessing
from proteingym_b200.tranception_engine import prior_rows
from proteingym_b200.trancepteve_engine import iterative_recalibrations, retrieval_weights


def _meta(name):
    return json.load(open(os.path.join(GOLDEN, name, "meta.json")))


@pytest.mark.parametrize("name", list(CASES))
def test_msa_processing_matches_reference(name, tmp_path):
    case, meta = CASES[name], _meta(name)
    inp = make_inputs(case, str(tmp_path), weights_file=os.path.join(GOLDEN, name, "msa_weights.npy"))
    m = MSAProcessing(inp["msa_file"], weights_location=inp["weights_file"], threshold_sequence_frac_gaps=case["seq_thr"],
                      threshold_focus_cols_frac_gaps=case["col_thr"])
    assert m.focus_cols == meta["focus_cols"] and m.seq_len == meta["focus_seq_len"]
    assert m.num_sequences == len(m.weights) == len(m.seq_name_to_weight)
    if case["kind"] == "TranceptEVE":
        assert m.num_sequences == meta["EVE_processed_depth"]
    assert "".join(m.focus_seq_trimmed) == "".join(meta["target_seq"][case["msa"][0] + c] for c in m.focus_cols)
    oh = m.one_hot_encoding
    assert oh.shape == (m.num_sequences, m.seq_len, 20) and np.all(oh.sum(-1) <= 1)


def test_msa_processing_error_paths(tmp_path):
    case = CASES["trancepteve_msa_only"]
    inp = make_inputs(case, str(tmp_path))
    with pytest.raises(SystemExit):  # the reference prints "Provided weights location is invalid" and exits (msa_utils.py:363-365)
        MSAProcessing(inp["msa_file"], weights_location=str(tmp_path / "missing.npy"))
    np.save(inp["weights_file"], np.ones(3))
    with pytest.raises(IndexError):  # fewer weights than retained sequences: weights[i] fails, as in the reference (:393)
        MSAProcessing(inp["msa_file"], weights_location=inp["weights_file"])
    with pytest.raises(AssertionError, match="Invalid fragment filtering parameter"):
        MSAProcessing(inp["msa_file"], use_weights=False, threshold_sequence_frac_gaps=1.5)


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c["kind"] == "TranceptEVE"])
def test_eve_log_prior_matches_reference_sampling(name, tmp_path):
    """Same generator seed, same draw order -> the reference's Monte-Carlo average bit for bit (CPU generator here); also the
    cache-file round trip in the reference's location and format."""
    case, meta = CASES[name], _meta(name)
    inp = make_inputs(case, str(tmp_path), weights_file=os.path.join(GOLDEN, name, "msa_weights.npy"))
    m = MSAProcessing(inp["msa_file"], weights_location=inp["weights_file"], threshold_sequence_frac_gaps=case["seq_thr"],
                      threshold_focus_cols_frac_gaps=case["col_thr"])
    paths = []
    for sd in case["eve_seeds"]:
        pth = os.path.join(inp["eve_dir"], f"TARGET_msa_seed_{sd}")
        torch.save({"model_state_dict": synth.make_eve_state(m.seq_len, seed=100 + sd)}, pth)
        paths.append(pth)
    ref = np.load(os.path.join(GOLDEN, name, "eve_log_prior_init.npy"))
    got = eve_prior.eve_log_prior(paths, inp["params_file"], m, case["L"], case["msa"][0], case["n_samples"], device="cpu").numpy()
    assert np.array_equal(np.isfinite(got), np.isfinite(ref))
    fin = np.isfinite(ref)
    assert np.abs(got[fin] - ref[fin]).max() < 1e-5
    for i, pth in enumerate(paths):  # cache written where the reference looks for it, readable as the reference reads it
        loc = eve_prior.cache_location(pth, case["n_samples"])
        assert loc == os.path.join(inp["eve_dir"], "log_prior", f"TARGET_msa_seed_{case['eve_seeds'][i]}_{case['n_samples']}_log_space")
        with open(loc, "rb") as fh:
            single = pickle.load(fh)
        one = np.load(os.path.join(GOLDEN, name, f"eve_log_prior_model{i}.npy"))
        assert np.abs(np.nan_to_num(single.numpy(), neginf=0) - np.nan_to_num(one, neginf=0)).max() < 1e-5
    again = eve_prior.eve_log_prior(paths, inp["params_file"], m, case["L"], case["msa"][0], case["n_samples"], device="cpu").numpy()
    assert np.array_equal(np.nan_to_num(again, neginf=0), np.nan_to_num(got, neginf=0))


def test_local_reparameterisation_sampler_has_the_reference_distribution():
    """eve_prior's batched sampler draws pre-activations instead of weights. Same distribution as the reference's weight-by-weight
    sampling: identical when the posterior variances vanish, and Monte-Carlo averages that agree as closely as two independent
    streams of the reference-order sampler agree with each other."""
    import copy
    P = copy.deepcopy(synth.EVE_TINY_PARAMS)
    P["decoder_parameters"]["hidden_layers_sizes"] = [24, 32, 60]   # alphabet | last hidden size
    assert eve_prior.local_sampling_supported(P["decoder_parameters"]) and not eve_prior.local_sampling_supported(synth.EVE_TINY_PARAMS["decoder_parameters"])
    L = 9
    focus, cols = list(synth.random_protein(L, 3)), list(range(L))
    st0 = synth.make_eve_state(L, P, seed=7, log_var=-80.0)
    st0["encoder.fc_log_var.bias"].fill_(-80.0)
    st0["encoder.fc_log_var.weight"].zero_()
    run = lambda st, n, how, seed=42: eve_prior.eve_log_prior_single(st, P, focus, cols, L, 0, n, device="cpu", sampler=how, seed=seed)  # noqa: E731
    a, b = run(st0, 3, "stream"), run(st0, 3, "local")
    fin = torch.isfinite(a)
    assert torch.equal(fin, torch.isfinite(b)) and (a[fin] - b[fin]).abs().max() < 1e-5
    st = synth.make_eve_state(L, P, seed=7, log_var=-3.0)
    n = 4000
    s1, s2, l1 = run(st, n, "stream"), run(st, n, "stream", 7), run(st, n, "local")
    big = run(st, 400000, "local", 11)                      # a near-exact answer is cheap with the batched sampler
    noise = (s1[fin] - s2[fin]).abs().mean().item()
    assert noise > 1e-3                                      # the sampling matters at this variance
    assert (l1[fin] - s1[fin]).abs().mean().item() < 1.5 * noise
    assert (s1[fin] - big[fin]).abs().mean().item() < noise and (l1[fin] - big[fin]).abs().mean().item() < noise
    with pytest.raises(ValueError):
        eve_prior.eve_log_prior_single(st, synth.EVE_TINY_PARAMS, focus, cols, L, 0, 3, device="cpu", sampler="local")


def test_retrieval_weight_ladder():
    """Depth thresholds of the constructor (trancepteve/model_pytorch.py:720-763)."""
    f = lambda m, e: retrieval_weights("TranceptEVE", "aggregate_substitution", m, e)  # noqa: E731
    assert [f(d, 0)[0] for d in (0, 9, 10, 99, 100, 999, 1000, 9999, 10000, 99999, 100000)] == [0.0, 0.0, 0.1, 0.1, 0.3, 0.3, 0.4, 0.4, 0.4, 0.4, 0.5]
    assert [f(0, d)[1] for d in (0, 9, 10, 99, 100, 999, 1000, 9999, 10000, 99999, 100000)] == [0.0, 0.0, 0.3, 0.3, 0.6, 0.6, 0.7, 0.7, 0.7, 0.7, 0.8]
    assert retrieval_weights("Tranception", "aggregate_substitution", 5, 5) == (0.6, 0.0)
    assert retrieval_weights("TranceptEVE", "aggregate_indel", 9, 500) == (0.0, 0.0)
    assert retrieval_weights("TranceptEVE", "aggregate_indel", 10, 0) == (0.5, 0.1)
    assert retrieval_weights("TranceptEVE", "aggregate_substitution", 5, 5, True, 0.25, 0.75) == (0.25, 0.75)
    for name in CASES:
        meta = _meta(name)
        got = retrieval_weights(CASES[name]["kind"], "aggregate_substitution", meta["MSA_processed_depth"], meta["EVE_processed_depth"])
        assert got == (meta["retrieval_inference_MSA_weight"], meta["retrieval_inference_EVE_weight"])


def test_prior_rows_index_arithmetic():
    T = 12
    # slice [4, 14) of the protein, MSA over [6, 11): 5 overlapping positions
    p = np.full(T, -1, np.int32)
    prior_rows(p, None, 4, 14, 6, 11, False)
    assert list(p) == [-1, -1, 6, 7, 8, 9, 10, -1, -1, -1, -1, -1]
    p = np.full(T, -1, np.int32)
    prior_rows(p, None, 4, 14, 6, 11, True)   # reversed sequence: offset max(0, we - msa_end) = 3, rows descending
    assert list(p) == [-1, -1, -1, 10, 9, 8, 7, 6, -1, -1, -1, -1]
    p = np.full(T, -1, np.int32)
    prior_rows(p, None, 0, 5, 6, 11, False)   # no overlap
    assert (p == -1).all()
    # non-focus rows 7 and 9: EVE index cleared; MSA row re-derived from (position + ws)
    nf = np.zeros(20, bool)
    nf[[7, 9]] = True
    p, q = np.full(T, -1, np.int32), np.full(T, -1, np.int32)
    prior_rows(p, q, 4, 14, 6, 11, False, nf)
    assert list(p) == [-1, -1, 6, 7, 8, 9, 10, -1, -1, -1, -1, -1] and list(q) == [-1, -1, 6, -1, 8, -1, 10, -1, -1, -1, -1, -1]
    p, q = np.full(T, -1, np.int32), np.full(T, -1, np.int32)
    prior_rows(p, q, 4, 14, 6, 11, True, nf)
    # flipped: position 4 holds row 9 -> the reference maps it to protein coordinate 4 + 4 = 8 -> slice index 2 of the reversed
    # slice -> row 8; position 6 holds row 7 -> coordinate 10 -> slice index 4 -> row 6
    assert list(q) == [-1, -1, -1, 10, -1, 8, -1, 6, -1, -1, -1, -1]
    assert list(p) == [-1, -1, -1, 10, 8, 8, 6, 6, -1, -1, -1, -1]
    # window ending beyond the MSA on a flipped sequence: a non-focus position can land outside the MSA -> (1 - alpha) only
    nf = np.zeros(40, bool)
    nf[12] = True
    p, q = np.full(30, -1, np.int32), np.full(30, -1, np.int32)
    prior_rows(p, q, 10, 30, 0, 14, True, nf)  # lo, hi = 10, 14; a0 = 16; row 12 sits at position 17 -> coordinate 27 >= 14
    assert p[17] == -2 and q[17] == -1 and list(p[16:20]) == [13, -2, 11, 10]


def test_iterative_recalibration_reaches_target():
    g = torch.Generator().manual_seed(0)
    x = torch.log_softmax(3 * torch.randn((40, 20), generator=g), dim=-1)
    target = x.mean() * 0.7
    y = iterative_recalibrations(x, target)
    assert abs(y.mean() - target) <= 1e-3 and torch.allclose(torch.logsumexp(y, -1), torch.zeros(40), atol=1e-5)
    assert iterative_recalibrations(x, x.mean()) is x  # already there: untouched


@pytest.mark.parametrize("name", ["trancepteve_nonfocus", "trancepteve_long"])
def test_host_logic_reproduces_reference_scores(name, tmp_path):
    """Recalibration + fused scoring through TranceptEVEScorer's own code paths, CPU forward underneath, against the reference
    class's score_mutants output. (The other two cases run on the GPU in test_gpu_trancepteve.py.)"""
    from cpu_trancepteve import CpuTranceptEVE
    case, meta = CASES[name], _meta(name)
    gd = os.path.join(GOLDEN, name)
    a = case["arch"]
    arch = synth.TranceptionArch(a[0], a[1], a[2], a[3], n_ctx=a[4])
    st = synth.make_tranception_state(arch, meta["tranception_seed"])
    inp = make_inputs(case, str(tmp_path))
    eve = np.load(os.path.join(gd, "eve_log_prior_init.npy")) if case["kind"] == "TranceptEVE" else None
    sc = CpuTranceptEVE(arch, st, meta["target_seq"], case["kind"], np.load(os.path.join(gd, "msa_log_prior_init.npy")), eve,
                        case["msa"][0], case["msa"][1], (meta["MSA_processed_depth"], meta["EVE_processed_depth"]), meta["focus_cols"],
                        case["col_thr"], case["msa_recal"], case["eve_recal"])
    rows, labels = sc.get_transformer_log_softmax(meta["target_seq"])
    assert list(labels) == meta["wt_shift_labels"]
    assert np.abs(rows.numpy() - np.load(os.path.join(gd, "wt_log_softmax_msa_fused.npy"))).max() < 1e-4
    out = sc.score_mutants(inp["dms"], meta["target_seq"])
    ref = pd.read_csv(os.path.join(gd, "reference_scores.csv"))
    assert list(out.columns) == list(ref.columns) and list(out["mutated_sequence"]) == list(ref["mutated_sequence"])
    for c in ("avg_score_L_to_R", "avg_score_R_to_L", "avg_score"):
        assert np.abs(out[c].values - ref[c].values).max() < 2e-5, c
    assert list(out["mutant"]) == list(ref["mutant"])
    for mine, fn in ((sc.MSA_log_prior, "msa_log_prior_final.npy"), (sc.EVE_log_prior, "eve_log_prior_final.npy")):
        want = np.load(os.path.join(gd, fn))
        assert np.array_equal(np.isfinite(mine.numpy()), np.isfinite(want))
        assert np.abs(np.nan_to_num(mine.numpy(), neginf=0) - np.nan_to_num(want, neginf=0)).max() < 1e-4


@pytest.mark.parametrize("tag", ["tranception", "trancepteve"])
def test_cli_flag_surface_matches_reference(tag):
    """tests/golden/<tag>_cli_flags.json: the reference parser's actions, dumped by oracle/gen_golden_trancepteve.py cli."""
    from proteingym_b200 import score_trancepteve, score_tranception_proteingym
    parser = {"tranception": score_tranception_proteingym, "trancepteve": score_trancepteve}[tag].create_parser()
    mine = {}
    for a in parser._actions:
        if not a.option_strings or a.dest == "help":
            continue
        mine[a.dest] = {"opts": sorted(a.option_strings), "default": str(a.default), "nargs": str(a.nargs),
                        "type": getattr(a.type, "__name__", str(a.type)), "choices": list(a.choices) if a.choices else None,
                        "const": str(a.const)}
    ref = json.load(open(os.path.join(GOLDEN, tag + "_cli_flags.json")))
    assert set(mine) - set(ref) <= {"precision", "device", "MSA_log_prior_npy", "EVE_sampler"} and not set(ref) - set(mine)
    for k, v in ref.items():
        assert mine[k] == v, k


def test_prefix_reuse_identity_and_policy_saving():
    """The identity behind exact wild-type-prefix reuse, checked with the oracle's CPU forward, and the row counts Tranception's reuse
    policy plans for a config-4-like assay (L = 512 single substitutions)."""
    from oracle import tranception_oracle as O
    from proteingym_b200.decoder import prefix_split
    from proteingym_b200.tranception_engine import TranceptionScorer, tokenize
    arch = synth.TranceptionArch(2, 128, 4, 256)
    st = synth.make_tranception_state(arch, 3)
    wt = synth.random_protein(40, 8)
    rows_wt, tot_wt = O.fused_logprob_rows(st, wt, arch.layers, arch.heads)
    for mut in ("A7C" if wt[6] == "A" else f"{wt[6]}7C", f"{wt[0]}1W:{wt[30]}31Y", f"{wt[39]}40D"):
        ms = synth.apply_mutant(wt, mut)
        for rev in (False, True):
            x, y = (ms[::-1], wt[::-1]) if rev else (ms, wt)
            rows_y, tot_y = O.fused_logprob_rows(st, y, arch.layers, arch.heads) if rev else (rows_wt, tot_wt)
            rows_x, tot_x = O.fused_logprob_rows(st, x, arch.layers, arch.heads)
            tx, ty = tokenize(x), tokenize(y)
            fd = next(i for i in range(len(tx)) if tx[i] != ty[i])
            assert np.abs(rows_x[:fd] - rows_y[:fd]).max() < 1e-6           # identical states before the first changed token
            tail = lambda r, t: sum(float(r[k, t[k + 1]]) for k in range(fd, len(t) - 1))  # noqa: E731
            delta = (float(rows_y[fd - 1, tx[fd]]) - float(rows_y[fd - 1, ty[fd]])) + tail(rows_x, tx) - tail(rows_y, ty)
            assert abs(delta - (tot_x - tot_y)) < 1e-4
    # the policy on a 512-residue protein with 400 random single substitutions, both directions
    seq = synth.random_protein(512, 1)
    muts = synth.sample_mutants(seq, 400, 2)
    df = pd.DataFrame({"mutant": muts, "mutated_sequence": [synth.apply_mutant(seq, m) for m in muts]})
    sc = TranceptionScorer.__new__(TranceptionScorer)
    sc.n_ctx = 1024
    sl = sc.slices(df, seq)
    is_mut = (sl["mutated_sequence"] != seq).to_numpy()
    tokens = rows_exact = rows_aligned = 0
    for rev in (False, True):
        strings = [s[::-1] if rev else s for s in sl["sliced_mutated_sequence"]]
        w = seq[::-1] if rev else seq
        rows, _, plain, groups = sc.reuse_policy(strings, list(zip(sl["window_start"], sl["window_end"])), [w if m else None for m in is_mut])
        assert rows[len(strings):] == [w] and list(groups) == [len(strings)]     # one window: one wild-type pass
        start = dict.fromkeys(plain, 0)
        start.update({r: s for s, members in groups[len(strings)].items() for r in members})
        mut = np.flatnonzero(is_mut)
        assert len(mut) == len(muts) and set(start) == set(range(len(strings)))
        assert all(len(strings[i]) + 2 == 514 for i in mut)
        fds = [prefix_split(strings[i], w, 1, 128)[0] for i in mut]
        tokens += 514 * len(mut)
        rows_exact += sum(514 - fd for fd in fds)
        rows_aligned += sum(514 - start[i] for i in mut)
        if not rev:
            i0 = int(np.flatnonzero(sl["mutated_sequence"] == synth.apply_mutant(seq, muts[0]))[0])
            assert fds[list(mut).index(i0)] == int(muts[0][1:-1])  # residue i (1-based) is token i
    exact, aligned = rows_exact / tokens, rows_aligned / tokens
    assert 0.45 < exact < 0.55 and 0.55 < aligned < 0.70   # half the rows exactly; ~5/8 with 128-row tile alignment
