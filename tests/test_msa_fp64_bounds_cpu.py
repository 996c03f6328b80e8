"""CPU: the bounds of tests/test_gpu_z_msa_fp64.py are tight enough to catch a kernel that loses precision inside an attention. The fp64
oracle is evaluated with one emulated fault (msa_oracle.FAULTS: the tied attention's q/k/v or P, or the column attention's q/k/v,
rounded to fp16 with the lo plane dropped) on every case of that file; the GPU test fails when any case exceeds its mode's bound, so
each fault must exceed twice the f16x3 and the f16f8 bound on some case. The ablated states must also isolate the attention they keep."""
import functools

import pytest

from msa_fp64_cases import BOUND, CASES, max_err
from oracle import msa_oracle as MO

TIED = ("tied_qkv_f16", "tied_p_f16")


@functools.lru_cache(maxsize=None)
def exact(case):
    return case.reference()


@pytest.mark.parametrize("fault", MO.FAULTS)
def test_emulated_fault_exceeds_twice_the_bounds(fault):
    errs = {c: max_err(c.reference(fault), exact(c)) for c in CASES}
    print(f"\n{fault}: " + " ".join(f"{c.id}={e:.1e}" for c, e in errs.items()))
    for c, e in errs.items():
        # a state without the faulty attention does not see the fault (R = 1 has no column softmax: v -> out_proj)
        blind = c.state == ("column-only" if fault in TIED else "row-only") or (fault == "col_qkv_f16" and c.R == 1)
        assert (e == 0) == blind, (c.id, e)
    for mode in ("f16x3", "f16f8"):
        caught = [c.id for c, e in errs.items() if e >= 2 * BOUND[mode]]
        assert caught, f"{fault}: no case reaches twice the {mode} bound {BOUND[mode]:.0e} (largest {max(errs.values()):.2e})"
        print(f"{fault} exceeds 2 x the {mode} bound on {len(caught)} of {len(CASES)} cases")
