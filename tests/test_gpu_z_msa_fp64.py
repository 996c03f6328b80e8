"""GPU (-m gpu): pg_msa_masked_marginals against the fp64 oracle (oracle/msa_oracle.py) on the same seeded q/k-gain-1 models, at the
shapes where the MSA Transformer's data movement changes form: the Cp / Kp padding of the tied attention, long alignments, head counts
that are not whole warps, several alignments per pass, row positions, 1024-column windows, the pruned last layer alone and after a
general layer, and the three precision modes. States with one attention's output projection zeroed ("row-only", "column-only") tell
the two attentions apart. Cases and bounds: tests/msa_fp64_cases.py; tests/test_msa_fp64_bounds_cpu.py shows the bounds would catch a
kernel that dropped a lo plane."""
import functools

import pytest
import torch

from msa_fp64_cases import BOUND, CASES, MODES, Case, max_err

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def reference(case):
    return case.reference()


@pytest.mark.parametrize("precision", MODES)
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_masked_marginals_match_fp64(case, precision):
    sc = case.scorer(precision)
    try:
        got = sc.masked_marginal_rows(case.tokens(), case.cols()).cpu().numpy()
    finally:
        sc.close()
    err = max_err(got, reference(case))
    print(f"\nMSA fp64 {case.id} {precision}: max|dlogp|={err:.2e} (bound {BOUND[precision]:.0e})")
    assert err < BOUND[precision]


@pytest.mark.parametrize("precision", MODES)
def test_pass_split_and_rerun_are_bit_identical(precision):
    """Cw = 129 (Cp = 256: the tied GEMMs as CTA pairs): 14 positions as 14 passes of one alignment or 2 passes of 7 give the same
    bits, and so does a second call."""
    case = Case("cw129", C=129)
    toks, pos = case.tokens(), list(range(0, 129, 10)) + [128]
    one, seven = Case("cw129", C=129, per_pass=1).scorer(precision), Case("cw129", C=129, per_pass=7).scorer(precision)
    try:
        a, b = one.masked_marginal_rows(toks, pos), seven.masked_marginal_rows(toks, pos)
        again = seven.masked_marginal_rows(toks, pos)
    finally:
        one.close(); seven.close()
    assert len(pos) == 14
    assert torch.equal(a, b) and torch.equal(b, again)
