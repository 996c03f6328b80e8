"""CPU: the bounds of tests/test_gpu_tranception_fp64.py are tight enough to catch a Tranception kernel that loses precision or reads the
wrong data. The fp64 oracle is evaluated with one emulated fault (tranception_oracle.FAULTS: a dropped lo plane of the attention's
q/k/v or P or of the conv input, a lost conv halo at 64-row tiles, or the ALiBi slope indexed by conv group) on every case of that file
but the 36-layer one; the GPU test fails when any case exceeds its mode's bound, so each fault must exceed twice the f16x3 and the
f16f8 bound on some case. Two faults are invisible on part of the grid, and are asserted to be exactly so: with 4 heads every head
has the same slope, and a sequence of at most 64 tokens has no conv tile edge. They are why the grid has more than the 4-head model."""
import functools

import pytest

from oracle import tranception_oracle as TO
from tranception_fp64_cases import BOUND, CASES, max_err

CPU_CASES = [c for c in CASES if c.cpu]


@functools.lru_cache(maxsize=None)
def exact(case):
    return case.reference()


def _blind(fault, case):
    return ((fault == "alibi_slope_by_group" and case.heads == 4) or
            (fault == "conv_tile_edge" and max(case.lens) <= 64))


@pytest.mark.parametrize("fault", TO.FAULTS)
def test_emulated_fault_exceeds_twice_the_bounds(fault):
    errs = {c: max_err(c.reference(fault), exact(c)) for c in CPU_CASES}
    print(f"\n{fault}: " + " ".join(f"{c.id}={e:.1e}" for c, e in errs.items()))
    for c, e in errs.items():
        if _blind(fault, c):
            assert e == 0, (c.id, e)
    for mode in ("f16x3", "f16f8"):
        caught = [c.id for c, e in errs.items() if e >= 2 * BOUND[mode]]
        assert caught, f"{fault}: no case reaches twice the {mode} bound {BOUND[mode]:.0e} (largest {max(errs.values()):.2e})"
        print(f"{fault} exceeds 2 x the {mode} bound on {len(caught)} of {len(CPU_CASES)} cases")
