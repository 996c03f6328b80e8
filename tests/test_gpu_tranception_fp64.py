"""GPU (-m gpu): the Tranception decoder per token against the fp64 oracle (oracle/tranception_oracle.py) on the same seeded models:
every predicted row and vocabulary column, at 4, 12, 16 and 20 heads (one ALiBi slope per head group at 4 heads; the S, M and L
head groups otherwise), at the 64-row attention / conv tile edges, the conv halo rows, the 128-row prefix tile and n_ctx, in ragged
batches, at Tranception-L depth and with the retrieval fusions. Then the exact wild-type-prefix reuse (pg_ar_prefix_begin /
pg_ar_loglik_prefix): its rows are bit-identical to the plain path's; and the plain rows do not depend on how the sequences are
split into passes, also when one pass holds more than 65 535 sequences. Cases and bounds: tests/tranception_fp64_cases.py;
tests/test_tranception_fp64_bounds_cpu.py shows the bounds would catch an emulated kernel fault."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from oracle import tranception_oracle as TO
from proteingym_b200 import _lib, synth
from proteingym_b200 import tranception_engine as TE
from tranception_fp64_cases import BOUND, BY_ID, CASES, MODES, Case, label_sums, max_err, model_state

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def reference(case):
    return case.reference()


@pytest.mark.parametrize("precision", MODES)
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_rows_match_fp64(case, precision):
    sc = case.scorer(precision)
    try:
        sums, rows = case.run(sc)
    finally:
        sc.close()
    ref = reference(case)
    assert [r.shape for r in rows] == [r.shape for r in ref]
    err = max_err(rows, ref)
    n_pred = np.asarray(case.lens) - 1
    sum_err = np.abs(sums.astype(np.float64) - label_sums(case, ref))
    print(f"\nTranception fp64 {case.id} {precision}: max|dlogp|={err:.2e} (bound {BOUND[precision]:.1e}), "
          f"max|dsum|/rows={float((sum_err / n_pred).max()):.2e}")
    assert err < BOUND[precision]
    assert (sum_err <= n_pred * BOUND[precision]).all(), sum_err


# ------------------------------------------------------------------------------------------------ exact wild-type-prefix reuse
PRIOR_KW = dict(alpha=float(np.float32(0.6)), msa_start=30)
# (heads, wild-type tokens T, starts): a 2-row suffix, a 1-row suffix (no predicted row of its own), a 44-row suffix, three
# starts in one window, and n_ctx with the suffix's last tile holding the 0.5-slope keys near 1023
PREFIX = [(12, 130, (128,)), (12, 257, (256,)), (12, 300, (256,)), (12, 422, (128, 256, 384)), (20, 1024, (896,))]


@functools.lru_cache(maxsize=None)
def reference_rows(heads, seqs):
    return TO.logprob_rows(model_state(2, heads), seqs, 2, heads)


def _mutate(seq, pos):
    c = seq[pos]
    return seq[:pos] + ("A" if c != "A" else "C") + seq[pos + 1:]


def _prefix_members(wt, start):
    """Strings that share tokens 0 .. start-1 with [CLS] wt [SEP]: the wild type itself and mutants whose first change is token
    start, start + 1 or the last residue (character = token - 1)."""
    T = len(wt) + 2
    toks = sorted({t for t in (start, start + 1, T - 2) if start <= t <= T - 2})
    return [wt] + [_mutate(wt, t - 1) for t in toks]


def _prow(seq, prior):
    pr = np.full(len(seq) + 2, -1, dtype=np.int32)
    TE.prior_rows(pr, None, 0, len(seq), PRIOR_KW["msa_start"], prior.shape[0] - 20, False)
    return pr


def _fusion(prior, prow, out_rows, keep):
    f = _lib.PgArFusion()
    f.alpha = PRIOR_KW["alpha"]
    if prior is not None:
        keep += [torch.from_numpy(prior).cuda(), torch.from_numpy(np.ascontiguousarray(prow)).cuda()]
        f.log_prior, f.prior_row = keep[-2].data_ptr(), keep[-1].data_ptr()
    f.out_logprobs = out_rows.data_ptr()
    return f


def _plain(sc, seqs, prior):
    kw = {} if prior is None else dict(prior=prior, windows=[(0, len(s)) for s in seqs], msa_end=prior.shape[0] - 20, **PRIOR_KW)
    return sc.sequence_logprobs(seqs, return_rows=True, **kw)


def _prefix_rows(sc, wt, seqs, start, prior):
    """pg_ar_prefix_begin on wt, then ONE pg_ar_loglik_prefix call on the suffixes (rows start ..) of seqs, which may be ragged
    -> (wild-type fused rows [T-1, V], per sequence its suffix rows [len - 1 - start, V], suffix sums)."""
    T = len(wt) + 2
    keep = []
    wt_ids = torch.from_numpy(TE.tokenize_batch([wt], T)[0]).cuda()
    wt_rows = torch.zeros((T, sc.vocab), device="cuda")
    tok = torch.zeros(T, device="cuda")
    f = _fusion(prior, _prow(wt, prior) if prior is not None else None, wt_rows, keep)
    _lib.check(sc.lib.pg_ar_prefix_begin(sc.handle, wt_ids.data_ptr(), T, C.byref(f), tok.data_ptr(), None), sc.handle)
    Tf = max(len(s) for s in seqs) + 2
    ids, lens = TE.tokenize_batch(seqs, Tf)
    Ts = Tf - start
    sfx_ids = torch.from_numpy(np.ascontiguousarray(ids[:, start:])).cuda()
    sfx_lens = torch.from_numpy(lens - start).cuda()
    rows = torch.zeros((len(seqs), Ts, sc.vocab), device="cuda")
    prow = np.stack([np.pad(_prow(s, prior), (0, Tf - len(s) - 2), constant_values=-1)[start:] for s in seqs]) if prior is not None else None
    f = _fusion(prior, prow, rows, keep)
    out = torch.zeros(len(seqs), device="cuda")
    _lib.check(sc.lib.pg_ar_loglik_prefix(sc.handle, sfx_ids.data_ptr(), sfx_lens.data_ptr(), len(seqs), Ts, start, C.byref(f),
                                          out.data_ptr(), None), sc.handle)
    torch.cuda.synchronize()
    rows = rows.cpu().numpy()
    return wt_rows.cpu().numpy()[:T - 1], [rows[b, :lens[b] - 1 - start] for b in range(len(seqs))], out.cpu().numpy()


@pytest.mark.parametrize("precision", MODES)
@pytest.mark.parametrize("with_prior", [False, True], ids=["plain", "prior"])
@pytest.mark.parametrize("heads,T,starts", PREFIX, ids=[f"h{h}-t{T}" for h, T, _ in PREFIX])
def test_prefix_rows_are_the_plain_rows(heads, T, starts, with_prior, precision):
    case = Case(f"h{heads}-prefix", heads, (T,))
    wt = synth.random_protein(T - 2, 31 * T)
    prior = np.log(np.random.RandomState(T).dirichlet(np.ones(25), size=T - 2)).astype(np.float32) if with_prior else None
    sc = case.scorer(precision)
    worst = 0.0
    try:
        for start in starts:
            members = _prefix_members(wt, start)
            _, plain = _plain(sc, members, prior)
            wt_rows, sfx, sfx_sums = _prefix_rows(sc, wt, members, start, prior)
            assert np.array_equal(wt_rows, plain[0])
            for m, p, s in zip(members, plain, sfx):
                assert s.shape == p[start:].shape and np.array_equal(s, p[start:]), (start, m == wt)
            # suffix sums: the plain rows' label terms from row start on (fp32 warp sums of the same values)
            lab = [np.asarray(TO.tokenize(m)[1:]) for m in members]
            want = [float(p[np.arange(len(l)), l][start:].astype(np.float64).sum()) for p, l in zip(plain, lab)]
            assert np.allclose(sfx_sums, want, rtol=0, atol=1e-5 * T)
            # ragged: the same call with truncated copies (lens[b] < Ts)
            if T - start > 2:
                rag = [members[-1], members[0][:start + (T - start) // 2 - 2], members[0][:start - 1]]
                _, plain_r = _plain(sc, rag, prior)
                _, sfx_r, _ = _prefix_rows(sc, wt, rag, start, prior)
                for p, s in zip(plain_r, sfx_r):
                    assert np.array_equal(s, p[start:])
            # against fp64 (unfused rows; the prior fusion is checked against fp64 by the fusion cases)
            if prior is None:
                worst = max(worst, max_err(plain, reference_rows(heads, tuple(members))))
    finally:
        sc.close()
    if prior is None:
        print(f"\nTranception prefix h{heads} T={T} {precision}: max|dlogp|={worst:.2e} (bound {BOUND[precision]:.1e})")
        assert worst < BOUND[precision]


@pytest.mark.parametrize("precision", ["f16x3", "f16"])
@pytest.mark.parametrize("with_prior", [False, True], ids=["plain", "prior"])
def test_reuse_sums_equal_plain_sums(with_prior, precision):
    """The engine's recombined sums (wild-type rows before `start` + suffix sums) equal the plain sums to fp32 rounding."""
    case = Case("h12-reuse", 12, (422,))
    wt = synth.random_protein(420, 5)
    muts = [_mutate(wt, p) for p in (126, 127, 128, 200, 254, 255, 256, 300, 382, 383, 384, 419)]
    muts.append(_mutate(_mutate(wt, 400), 130))
    prior = np.log(np.random.RandomState(3).dirichlet(np.ones(25), size=420)).astype(np.float32) if with_prior else None
    kw = dict(prior=prior, msa_end=400, **PRIOR_KW) if with_prior else {}
    sc = case.scorer(precision)
    try:
        got = sc._logprobs_with_reuse(muts, [(0, 420)] * len(muts), [wt] * len(muts), False, kw)
        full, run = sc.reuse_rows
        plain, rows = sc.sequence_logprobs(muts, windows=[(0, 420)] * len(muts), return_rows=True, **kw)
    finally:
        sc.close()
    assert run < full
    for g, p, r, m in zip(got, plain, rows, muts):
        lab = np.asarray(TO.tokenize(m)[1:])
        terms = r[np.arange(len(lab)), lab].astype(np.float64)
        tol = 2 * (len(lab) / 32 + 6) * 2.0 ** -24 * np.abs(terms).sum()
        assert abs(float(g) - float(p)) <= tol, (g, p, tol)


@pytest.mark.parametrize("precision", MODES)
def test_pass_split_is_bit_identical(precision):
    """The ragged 12-head batch as one pass, and as one sequence per pass (max_rows = the longest sequence's tokens)."""
    case = BY_ID["h12-ragged"]
    one = case.scorer(precision)
    split = case.scorer(precision, max_rows=max(case.lens))
    try:
        a_sums, a = case.run(one)
        b_sums, b = case.run(split)
    finally:
        one.close()
        split.close()
    assert np.array_equal(a_sums, b_sums)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("precision", ["f16x3", "f16"])  # the two-plane and the one-plane instance of the depthwise conv
def test_one_pass_over_65535_sequences(precision):
    """65 600 sequences of two and three tokens on the 4-head model as ONE pass (no kernel of the pass may depend on a 16-bit
    grid dimension for the sequence index), against the same sequences in three passes of under 30 000."""
    aa = "ACDEFGHIKLMNPQRSTVWY"
    seqs = [aa[i % 20] if i % 3 else "" for i in range(65600)]
    case = BY_ID["h4-t3"]
    one = case.scorer(precision, max_rows=1 << 18)
    split = case.scorer(precision, max_rows=90000)  # 30 000 sequences of T = 3 rows
    try:
        a_sums, a = one.sequence_logprobs(seqs, chunk_rows=1 << 18, return_rows=True)
        b_sums, b = split.sequence_logprobs(seqs, chunk_rows=1 << 18, return_rows=True)
    finally:
        one.close()
        split.close()
    assert np.isfinite(a_sums).all() and len(set(a_sums.tolist())) > 1
    assert np.array_equal(a_sums, b_sums)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
