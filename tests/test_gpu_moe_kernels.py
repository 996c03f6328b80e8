"""GPU: the ragged grouped form of the GEMM (ProGen3's experts) through pg_gemm_form, against fp64 of the operand planes the kernel reads:
expert segments of 0, 1, 77, 130 and 256 rows padded to 128 or 256, W blocks wider than N, an N that is not a multiple of 128, epilogues 0
(fp16 hi / lo), 8 (SiLU), 5 (SwiGLU) and 9 (fp32 store); tiles past the table's count must leave their rows untouched, and the two-CTA
form (256-row segments) must give the single-CTA form's bits."""
import ctypes as C

import numpy as np
import pytest
import torch

from proteingym_b200 import _lib

pytestmark = pytest.mark.gpu

COUNTS = [130, 0, 1, 256, 77]  # rows per expert
K, N, GB = 256, 192, 256       # reduction, output columns, W rows per expert (>= N)
# |out - fp64| / max |fp64| over the cases: about 4x the worst measured on an H100 80GB HBM3 at 700 W (nseg 1: 3.5e-4, most of it the
# fp16 rounding of the output; nseg 3: 1.0e-6)
BOUND = {1: 1.4e-3, 3: 4e-6}


def pack(w, nseg):
    n, k = w.shape
    out = torch.empty((n, k * (1 if nseg == 1 else 2)), dtype=torch.float16, device="cuda")
    _lib.check(_lib.load().pg_pack_weight(w.data_ptr(), n, k, 0 if nseg == 1 else 1, out.data_ptr(), None, None))
    return out


def planes(x, nseg):
    """fp32 rows -> fp16 operand rows [hi | lo] and the value the kernel reads (fp64)."""
    hi = x.half()
    if nseg == 1:
        return hi, hi.double()
    lo = (x - hi.float()).half()
    return torch.cat([hi, lo], dim=1), hi.double() + lo.double()


def layout(pad):
    """-> (expert of every tile, rows in use) for COUNTS padded to `pad`."""
    tiles = []
    for e, c in enumerate(COUNTS):
        tiles += [e] * ((c + pad - 1) // pad)
    return tiles, len(tiles) * pad


def run(nseg, epi, pad, cta2=1, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    E = len(COUNTS)
    tiles, used = layout(pad)
    M = used + 2 * pad  # two tiles past the table's count
    x = torch.randn((M, K), device="cuda", generator=g)
    w = torch.randn((E * GB, K), device="cuda", generator=g) / K ** 0.5
    a, av = planes(x, nseg)
    wp = pack(w, nseg)
    wv = wp[:, :K].double() + (wp[:, K:].double() if nseg == 3 else 0)
    t_exp = torch.tensor(tiles + [0, 0], dtype=torch.int32, device="cuda")
    t_cnt = torch.tensor([len(tiles)], dtype=torch.int32, device="cuda")
    args = _lib.PgGemmArgs()
    args.a, args.lda, args.w, args.ldw = a.data_ptr(), a.shape[1], wp.data_ptr(), wp.shape[1]
    args.M, args.N, args.K, args.nseg, args.epi = M, N, K, nseg, epi
    args.grp_rows_b = GB
    n_out = N // 2 if epi == 5 else N
    if epi == 9:
        out = torch.full((M, N), float("nan"), device="cuda")
        args.resid, args.ldr = out.data_ptr(), N
    else:
        fmt = 1 if nseg == 3 else 0
        out = torch.full((M, n_out * (2 if fmt else 1)), float("nan"), device="cuda", dtype=torch.float16)
        args.out_h, args.ldo, args.out_lo_off, args.out_fmt = out.data_ptr(), out.shape[1], (n_out if fmt else 0), fmt
    f = _lib.PgGemmForm()
    f.rg_expert, f.rg_tiles, f.rg_pad, f.rg_experts = t_exp.data_ptr(), t_cnt.data_ptr(), pad, E
    lib = _lib.load()
    _lib.check(lib.pg_set_tuning(b"gemm_cta2", cta2))
    try:
        _lib.check(lib.pg_gemm_form(C.byref(args), C.byref(f), None))
        torch.cuda.synchronize()
    finally:
        _lib.check(lib.pg_set_tuning(b"gemm_cta2", 1))
    ref = torch.full((M, n_out), float("nan"), dtype=torch.float64, device="cuda")
    for m, e in enumerate(tiles):
        acc = av[m * pad:(m + 1) * pad] @ wv[e * GB:e * GB + N].T
        if epi == 8:
            acc = acc * torch.sigmoid(acc)
        elif epi == 5:
            v = acc.view(pad, -1, 2, 8)
            acc = (torch.nn.functional.silu(v[:, :, 0]) * v[:, :, 1]).reshape(pad, -1)
        ref[m * pad:(m + 1) * pad] = acc
    got = out.double() if epi == 9 else out[:, :n_out].double() + (out[:, n_out:].double() if out.shape[1] > n_out else 0)
    return got, ref, used, out


@pytest.mark.parametrize("pad", [128, 256])
@pytest.mark.parametrize("nseg", [1, 3])
@pytest.mark.parametrize("epi", [0, 8, 5, 9])
def test_ragged_grouped_gemm_vs_fp64(epi, nseg, pad):
    got, ref, used, out = run(nseg, epi, pad)
    err = ((got[:used] - ref[:used]).abs().max() / ref[:used].abs().max()).item()
    print(f"\nragged epi {epi} nseg {nseg} pad {pad}: max |err| / max |ref| = {err:.2e}")
    assert np.isfinite(err) and err < BOUND[nseg]
    assert torch.isnan(out[used:].float()).all()  # tiles past the count are not computed


@pytest.mark.parametrize("epi", [0, 9])
def test_two_cta_form_is_bit_identical(epi):
    a, _, used, _ = run(3, epi, 256, cta2=1, seed=2)
    b, _, _, _ = run(3, epi, 256, cta2=0, seed=2)
    assert torch.equal(a[:used], b[:used])
