"""GPU (-m gpu): the row kernels between the GEMMs and the attention, kernel by kernel through their own entry points, against fp64
evaluations of the exact planes each kernel reads: the ESM embedding (K1), the LayerNorm forms (K2: padded planes, the column
permutation, the delta-operand base), the single-query attention of the pruned last ESM layer, ESM C's q/k LayerNorm + rotary, the
ESM-family LM head (K5), the autoregressive head with its retrieval fusion and sequence sums, and the combine of the fused 50 257-way
LM head.

Inputs are adversarial: a wrong rule (a token-dropout denominator, a fused column, a query row, a rotary sign, a dropped bias) moves
the result by far more than the bound. Output buffers start as NaN / 0xFF, so bytes a kernel leaves unwritten, or writes past its rows,
show up; where a path only moves bytes (permuted rows, untouched columns, zero padding, ignored targets) the test asks for
bit-identity. Every test prints its measured error next to its bound."""
import ctypes as C
import math

import pytest
import torch

from proteingym_b200 import _lib
from test_gpu_parity import q8, unpack_f8

pytestmark = pytest.mark.gpu
S8 = 4.0          # e4m3 scale of fmt 2 outputs
MASK_IDX = 32     # ESM <mask>
PG_ERR_ARG, PG_ERR_UNSUPPORTED = 1, 4
EPS = 2.0 ** -24  # fp32 unit roundoff


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def report(name, err, bound):
    print(f"\n[row kernels] {name}: max|err| = {err:.3e} (bound {bound:.3e})")
    assert err < bound, (name, err, bound)


def maxerr(a, b):
    """max |a - b| with NaN counted as inf: a NaN must not vanish in a later max()"""
    return torch.nan_to_num((a - b).abs(), nan=math.inf).max().item()


def i32(v):
    return torch.as_tensor(v, dtype=torch.int32).cuda()


def ptr(t):
    return t.data_ptr() if t is not None else None


def ln64(x, g=None, b=None):
    x = x.double()
    y = (x - x.mean(-1, keepdim=True)) / torch.sqrt(x.var(-1, unbiased=False, keepdim=True) + 1e-5)
    if g is not None:
        y = y * g.double()
    if b is not None:
        y = y + b.double()
    return y


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ------------------------------------------------------------------------------------------------ K1: ESM embedding
def run_embed(tokens, positions, win_start, P, T, d, E, pos, lnb, td, p_off, force):
    lib = _lib.load()
    x = torch.full((P * T + 1, d), float("nan"), device="cuda")  # one spare row: must stay NaN
    a = _lib.PgEsmEmbedArgs(tokens=ptr(tokens), n_tokens=tokens.numel(), positions=ptr(positions), win_start=ptr(win_start),
                            P=P, T=T, d=d, embed=ptr(E), pos_table=ptr(pos), lnb_gamma=ptr(lnb[0]) if lnb else None,
                            lnb_beta=ptr(lnb[1]) if lnb else None, token_dropout=td, mask_idx=MASK_IDX, p_offset=p_off,
                            force_mask_scale=force, x=x.data_ptr())
    _lib.check(lib.pg_esm_embed(C.byref(a), None))
    torch.cuda.synchronize()
    assert torch.isnan(x[-1]).all()
    return x[:-1]


def embed_ref(tokens, positions, win_start, P, T, E, pos, lnb, td, p_off, force):
    """fp64 of esm1.py:123-139 / esm2.py:83-94 for one masked copy per row p: x = embed(tok) with the masked token zeroed, times
    (1 - 0.15 * 0.8) / (1 - n_mask / T) (n_mask = 1 when the mask lies in the window, or under force_mask_scale), + pos[t + 2]."""
    tok = tokens.tolist()
    pos_l = positions.tolist() if positions is not None else [-1] * (p_off + P)
    ws_l = win_start.tolist() if win_start is not None else [0] * (p_off + P)
    idx, masked, scales = [], [], []
    for p in range(P):
        ws, mpos = ws_l[p_off + p], pos_l[p_off + p]
        has_mask = ws <= mpos < ws + T or force
        scales.append((1 - 0.15 * 0.8) / (1 - (1.0 / T if has_mask else 0.0)))
        for gi in range(ws, ws + T):
            masked.append(gi == mpos)
            idx.append(MASK_IDX if gi == mpos else tok[min(gi, len(tok) - 1)])
    m = torch.tensor(masked, device="cuda")
    x = E.double()[torch.tensor(idx, device="cuda")]
    if td:
        x = x.masked_fill(m[:, None], 0.0) * torch.tensor(scales, device="cuda", dtype=torch.float64).repeat_interleave(T)[:, None]
    if pos is not None:
        x = x + pos.double()[2:T + 2].repeat(P, 1)
    if lnb:
        x = ln64(x, *lnb)
    return x


# ESM-1v (token dropout, learned positions), ESM2 (token dropout, rotary: no position table), ESM-1b (learned positions,
# emb_layer_norm_before, no token dropout), and token dropout under LayerNorm-before
EMBED_KINDS = {"esm1v": (1, True, False), "esm2": (1, False, False), "esm1b": (0, True, True), "td+lnb": (1, True, True)}
# fp32 error model: the rescale factor takes three roundings (1/T, 1 - ratio, the quotient), then the product and the position add one
# each: <= 5 * 2^-24 * max|x| (measured 1.4 * 2^-24 on an H100 80GB HBM3 at 700 W). Under LayerNorm-before, the centred values of
# a row whose mean is ~10 std away from zero lose 2^-24 |mean| each, ~10 ulp of the output: 48 * 2^-24 * max|y| (measured 13.8).
EMBED_BOUND = {False: 5 * EPS, True: 48 * EPS}


@pytest.mark.parametrize("T", [3, 4, 8, 1026])
@pytest.mark.parametrize("kind", list(EMBED_KINDS))
def test_esm_embed_matches_fp64(kind, T):
    """Masked copies at the first, last and a middle token of plain and shifted windows, a copy without a mask (positions = -1), masks
    outside their window on either side, windows that run past the last token, p_offset > 0 (entries before it would move every copy),
    and the same copies under force_mask_scale. At T = 3 and 4 a denominator of T - 2 instead of T is infinite or doubles the rescale."""
    td, has_pos, has_lnb = EMBED_KINDS[kind]
    d = 320
    g = gen(T * 7 + len(kind))
    E = torch.randn(33, d, device="cuda", generator=g) * 2
    pos = torch.randn(T + 2, d, device="cuda", generator=g) if has_pos else None
    lnb = (torch.randn(d, device="cuda", generator=g), torch.randn(d, device="cuda", generator=g)) if has_lnb else None
    if has_lnb:
        E = E + 20.0  # rows ~10 std off zero: one-pass statistics would not hold the bound
    n_tokens = T + 4
    tokens = torch.randint(4, 29, (n_tokens,), device="cuda", generator=g, dtype=torch.int32)
    copies = [(5, 6), (5, 5),  # before p_offset: never read
              (0, 0), (0, T - 1), (0, T // 2), (0, -1), (3, 3), (3, 3 + T - 1), (3, 1), (4, 4 + T + 1), (7, 7 + T // 2)]
    p_off = 2
    ws = i32([c[0] for c in copies])
    mp = i32([c[1] for c in copies])
    P = len(copies) - p_off
    worst = bound = 0.0
    for force in (0, 1):
        got = run_embed(tokens, mp, ws, P, T, d, E, pos, lnb, td, p_off, force).double()
        ref = embed_ref(tokens, mp, ws, P, T, E, pos, lnb, td, p_off, force)
        worst = max(worst, maxerr(got, ref))
        bound = max(bound, EMBED_BOUND[has_lnb] * ref.abs().max().item())
    # no positions / win_start arrays at all: every copy is unmasked and starts at token 0
    got = run_embed(tokens, None, None, 2, T, d, E, pos, lnb, td, 0, 0).double()
    ref = embed_ref(tokens, None, None, 2, T, E, pos, lnb, td, 0, 0)
    worst = max(worst, maxerr(got, ref))
    report(f"embed {kind} T={T}", worst, bound)


# ------------------------------------------------------------------------------------------------ K2: LayerNorm forms
def ln_out_buffer(rows, dp, fmt):
    """Output rows of width W (+ 4 guard columns that must stay 0xFF): fmt 0 [hi (dp)], 1 [hi | lo], 2 [hi | lo8 (dp B) | hi8 (dp B)]."""
    W = dp if fmt == 0 else 2 * dp
    ldo = W + 4
    return torch.full((rows, 2 * ldo), 0xFF, device="cuda", dtype=torch.uint8), W, ldo


def run_ln(x, g, b, d, fmt, dp=0, perm=(0, 0), base=None, base_T=0, expect=0):
    lib = _lib.load()
    rows = x.shape[0]
    out, W, ldo = ln_out_buffer(rows, max(dp, d), fmt)
    f = _lib.PgLnForm(dp=dp, perm_R=perm[0], perm_C=perm[1], base=ptr(base), base_T=base_T)
    rc = lib.pg_layernorm_form(x.data_ptr(), x.shape[1], g.data_ptr(), b.data_ptr(), rows, d, out.data_ptr(), ldo, max(dp, d) if fmt else 0,
                               fmt, S8 if fmt == 2 else 0.0, C.byref(f), None)
    if expect:
        assert rc == expect, (rc, lib.pg_last_error(None))
        torch.cuda.synchronize()
        assert (out == 0xFF).all()  # refused: nothing launched
        return None
    _lib.check(rc)
    torch.cuda.synchronize()
    assert (out[:, 2 * W:] == 0xFF).all()  # guard columns between rows
    return out


def ln_planes(out, dp, fmt):
    """-> (hi fp16 [rows, dp], the fp64 value hi (+ lo / lo8), raw bytes of every plane [rows, 2 * W])"""
    hi = out[:, :2 * dp].contiguous().view(torch.float16)
    if fmt == 0:
        return hi, hi.double()
    if fmt == 1:
        return hi, hi.double() + out[:, 2 * dp:4 * dp].contiguous().view(torch.float16).double()
    h, lo8, _ = unpack_f8(out[:, :4 * dp], dp, S8)
    return hi, h + lo8


# fp32 two-pass LayerNorm against fp64 of the planes' value (hi + lo): c * max|y| per format. The centred values lose 2^-24 |mean|
# each, so rows with mean 30 and std 3 carry ~10 ulp of the output (measured 9.4 * 2^-24 * max|y| with fmt 1 on an H100 80GB HBM3 at
# 700 W); fmt 0 is fp16 rounding, 2^-11 relative (measured 0.73 of it); fmt 2 carries the low part in e4m3, 4 significant bits of a
# residual <= 2^-11 |y|, so 2^-15 relative (measured 0.46 of it)
LN_BOUND = {0: 2.0 ** -11, 1: 32 * EPS, 2: 2.0 ** -15}
LN_DIMS = [64, 480, 512, 516, 1280, 1284, 2560, 2564, 5120]


@pytest.mark.parametrize("fmt", [0, 1, 2])
@pytest.mark.parametrize("d", LN_DIMS)
def test_layernorm_padded_planes_match_fp64(d, fmt):
    """Every LayerNorm instance (d up to 512, 1280, 2560, 5120, just past each) unpadded and padded to the next multiple of 64 (480 ->
    512 is ESM2 35M's row); columns [d, dp) are exactly zero in every plane, the fp16 hi plane does not depend on the padding or the
    format, and the hi8 plane is e4m3(hi * s)."""
    rows = 77  # not a multiple of the 8 rows (warps) of a block
    gg = gen(d * 3 + fmt)
    x = torch.randn(rows, d, device="cuda", generator=gg) * 3 + 30.0
    g, b = torch.randn(d, device="cuda", generator=gg), torch.randn(d, device="cuda", generator=gg)
    ref = ln64(x, g, b)
    worst, bound, his = 0.0, 0.0, []
    for dp in (d, (d + 63) // 64 * 64 if d % 64 else d + 64):
        out = run_ln(x, g, b, d, fmt, dp=dp if dp != d else 0)
        hi, val = ln_planes(out, dp, fmt)
        his.append(hi[:, :d])
        worst = max(worst, maxerr(val[:, :d], ref))
        bound = max(bound, LN_BOUND[fmt] * ref.abs().max().item())
        W = dp if fmt == 0 else 2 * dp
        planes = out[:, :2 * W].reshape(rows, -1, 2 * dp) if fmt < 2 else None
        if fmt < 2:  # fp16 planes: dp halves each
            assert (planes[:, :, 2 * d:] == 0).all(), "padding columns of an fp16 plane are not zero"
        else:
            assert (out[:, 2 * d:2 * dp] == 0).all(), "padding of the hi plane is not zero"
            assert (out[:, 2 * dp + d:3 * dp] == 0).all() and (out[:, 3 * dp + d:4 * dp] == 0).all(), "padding of an e4m3 plane"
            assert torch.equal(out[:, 3 * dp:3 * dp + d], q8(hi[:, :d].float() * S8))
    assert same_bits(his[0], his[1])
    report(f"layernorm d={d} fmt {fmt}", worst, bound)


@pytest.mark.parametrize("R", [1, 3, 64, 65])
@pytest.mark.parametrize("Ccols", [1, 3, 64, 65])
def test_layernorm_column_permutation_is_plain_rows_permuted(R, Ccols):
    """perm_C: input row (b, r, c) goes to output row (b, c, r), bit-identical to the plain launch's row; unpadded fp16 hi/lo and the
    padded e4m3 rows of ESM2-35M-wide layers."""
    B = 2
    rows = B * R * Ccols
    for d, dp, fmt in ((64, 0, 1), (480, 512, 2)):
        gg = gen(R * 100 + Ccols + d)
        x = torch.randn(rows, d, device="cuda", generator=gg) * 2 + 1
        g, b = torch.randn(d, device="cuda", generator=gg), torch.randn(d, device="cuda", generator=gg)
        plain = run_ln(x, g, b, d, fmt, dp=dp)
        perm = run_ln(x, g, b, d, fmt, dp=dp, perm=(R, Ccols))
        bb, r, c = torch.meshgrid(torch.arange(B), torch.arange(R), torch.arange(Ccols), indexing="ij")
        src = (bb * R * Ccols + r * Ccols + c).flatten().cuda()
        dst = (bb * Ccols * R + c * R + r).flatten().cuda()
        assert same_bits(perm[dst], plain[src]), (R, Ccols, d)
    print(f"\n[row kernels] layernorm perm R={R} C={Ccols}: bit-identical")


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("d", [64, 1280, 2560])
def test_layernorm_delta_base_matches_fp64(d, fmt):
    """base form (f16d): out = LN(x) - base[row % base_T], formed in fp32 and rounded once. Rows are small perturbations of the base
    rows' own inputs, so the differences are small and a wrong base row is an O(1) error."""
    base_T, reps = 7, 5
    gg = gen(d + fmt)
    xb = torch.randn(base_T, d, device="cuda", generator=gg) * 2 + 3
    g, b = torch.randn(d, device="cuda", generator=gg), torch.randn(d, device="cuda", generator=gg)
    base = ln64(xb, g, b).half()
    x = xb.repeat(reps, 1) + 0.01 * torch.randn(base_T * reps, d, device="cuda", generator=gg)
    out = run_ln(x, g, b, d, fmt, base=base, base_T=base_T)
    _, val = ln_planes(out, d, fmt)
    ref = ln64(x, g, b) - base.double().repeat(reps, 1)
    # fp32 LayerNorm error on |LN(x)| (not on the small difference): rows with mean 3 and std 2 lose little in the centring (measured
    # 2.1 * 2^-24 * max|LN(x)| with fmt 1), then fp16 rounding of the difference for fmt 0
    ln_mag = ln64(x, g, b).abs().max().item()
    bound = 8 * EPS * ln_mag + (2.0 ** -11 * ref.abs().max().item() if fmt == 0 else 0.0)
    report(f"layernorm base d={d} fmt {fmt}", maxerr(val[:, :d], ref), bound)


def test_layernorm_refuses_bad_forms():
    """The forms the launcher refuses return PG_ERR_ARG / PG_ERR_UNSUPPORTED and launch nothing."""
    d = 64
    x = torch.randn(12, d + 4, device="cuda")
    g, b = torch.randn(d + 4, device="cuda"), torch.randn(d + 4, device="cuda")
    base = torch.zeros(3, d, device="cuda", dtype=torch.float16)
    run_ln(x, g, b, d, 1, perm=(2, 2), base=base, base_T=3, expect=PG_ERR_ARG)   # base + permutation
    run_ln(x, g, b, d, 1, dp=128, base=base, base_T=3, expect=PG_ERR_ARG)        # base + padding
    run_ln(x, g, b, d, 1, base=base, base_T=0, expect=PG_ERR_ARG)                # base without base_T
    run_ln(x, g, b, d, 1, perm=(5, 2), expect=PG_ERR_ARG)                         # 12 rows are not whole [5, 2] alignments
    run_ln(x, g, b, d, 1, perm=(0, 2), expect=PG_ERR_ARG)                         # perm_C without perm_R
    run_ln(x, g, b, d, 1, dp=62, expect=PG_ERR_ARG)                               # dp < d
    run_ln(x, g, b, d, 1, dp=66, expect=PG_ERR_ARG)                               # dp not a multiple of 4
    run_ln(x, g, b, 66, 1, expect=PG_ERR_ARG)                                     # d not a multiple of 4
    run_ln(x, g, b, d, 1, dp=-4, expect=PG_ERR_ARG)
    lib = _lib.load()
    out = torch.full((12, 4 * d), 0xFF, device="cuda", dtype=torch.uint8)
    f = _lib.PgLnForm()
    assert lib.pg_layernorm_form(x.data_ptr(), d, g.data_ptr(), b.data_ptr(), 12, d, out.data_ptr(), 2 * d, d, 2, 0.0, C.byref(f),
                                 None) == PG_ERR_ARG  # e4m3 planes without a scale
    big = torch.randn(2, 5124, device="cuda")
    gb = torch.ones(5124, device="cuda")
    outb = torch.full((2, 5124), 0xFF, device="cuda", dtype=torch.uint8)
    assert lib.pg_layernorm_form(big.data_ptr(), 5124, gb.data_ptr(), gb.data_ptr(), 2, 5124, outb.data_ptr(), 5124, 0, 0, 0.0,
                                 C.byref(f), None) == PG_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert (out == 0xFF).all() and (outb == 0xFF).all()


# ------------------------------------------------------------------------------------------------ single-query attention
MODES = [(1, 0), (3, 1), (3, 2)]  # (nseg, out_fmt)
MODE_IDS = ["nseg1", "nseg3-fmt1", "nseg3-fmt2"]


def peaked_qkv(B, T, H, row_sel, nseg, g):
    """q/k/v rows where the selected query row of every (sequence, head) scores one far key j* = (row_sel + T/2) % T about 10 above
    the rest: reading another query row, or dropping j*, moves the output by O(1)."""
    d = H * 64
    x = torch.randn(B * T, 3, H, 64, device="cuda", generator=g)
    x[:, 0] *= 0.1
    hot = []
    for b, r in enumerate(row_sel):
        j = (r + T // 2) % T
        hot.append(j)
        k = x[b * T + j, 1]
        x[b * T + r, 0] = 2.0 * k / k.norm(dim=-1, keepdim=True)  # score ~16 against j*, N(0, 4) against the rest
        x[b * T + j, 2] *= 3.0
    x = x.reshape(B * T, 3 * d)
    if nseg == 3:
        hi = x.half()
        op = torch.cat([hi, (x - hi.float()).half()], 1).contiguous()
        eff = hi.double() + op[:, 3 * d:].double()
    else:
        op = x.half().contiguous()
        eff = op.double()
    return op, eff, hot


def attn_out(rows, d, out_fmt):
    W = d if out_fmt == 0 else 2 * d
    return torch.full((rows, 2 * (W + 8)), 0xFF, device="cuda", dtype=torch.uint8), W + 8


def decode_rows(out, d, out_fmt):
    if out_fmt == 0:
        return out[:, :2 * d].contiguous().view(torch.float16).double()
    if out_fmt == 1:
        return out[:, :4 * d].contiguous().view(torch.float16).double().view(-1, 2, d).sum(1)
    hi, lo8, _ = unpack_f8(out[:, :4 * d], d, S8)
    return hi + lo8


def attn_args(op, out, ldo, B, T, H, nseg, out_fmt):
    d = H * 64
    a = _lib.PgAttnArgs()
    a.qkv, a.ld, a.lo_off = op.data_ptr(), op.shape[1], (3 * d if nseg == 3 else 0)
    a.out, a.ldo, a.out_lo_off = out.data_ptr(), ldo, (d if out_fmt else 0)
    a.B, a.T, a.heads, a.nseg = B, T, H, nseg
    a.out_fmt, a.out_scale = out_fmt, (S8 if out_fmt == 2 else 0.0)
    return a


# single fp16: the fp16 q/k/v rows are exact inputs, fp32 arithmetic, the output rounded to fp16 (2^-11 relative; measured 0.72 of the
# bound); x3: fp32 online softmax with __expf (relative error ~2^-21 at scores ~ +-20) on weights that sum to 1: ~2^-20 * max|v|
# (measured 0.68 of it at T = 1024); e4m3 low plane 2^-16 * max|out| on top (measured 0.67 of the sum). H100 80GB HBM3, 700 W.
def sq_bound(nseg, out_fmt, vmax, omax):
    if nseg == 1:
        return 2.0 ** -11 * omax + 2.0 ** -20 * vmax
    return 2.0 ** -20 * vmax + (2.0 ** -16 * omax if out_fmt == 2 else 0.0)


@pytest.mark.parametrize("T", [1, 2, 31, 32, 33, 64, 65, 514, 1024])
@pytest.mark.parametrize("nseg,out_fmt", MODES, ids=MODE_IDS)
def test_single_query_attention_matches_fp64_and_full_launch(nseg, out_fmt, T):
    """Row row_sel[b] (0, T - 1, a middle row) of every sequence against fp64 of the planes, and against the same row of a plain
    pg_attention launch over all rows; T below, at and above the 32 lanes that stride over the keys."""
    lib = _lib.load()
    B = 3
    row_sel = [0, T - 1, T // 2]
    worst = worst_full = bound = bound_full = 0.0
    for H in (1, 2, 20):
        d = H * 64
        op, eff, _ = peaked_qkv(B, T, H, row_sel, nseg, gen(T * 31 + H + nseg))
        out, ldo = attn_out(B + 1, d, out_fmt)
        a = attn_args(op, out, ldo, B, T, H, nseg, out_fmt)
        _lib.check(lib.pg_attention_rows(C.byref(a), i32(row_sel).data_ptr(), None))
        torch.cuda.synchronize()
        W = d if out_fmt == 0 else 2 * d
        assert (out[:, 2 * W:] == 0xFF).all() and (out[B] == 0xFF).all()  # guard columns and the row after the last
        got = decode_rows(out[:B], d, out_fmt)
        if out_fmt == 2:
            assert torch.equal(out[:B, 3 * d:4 * d], q8(out[:B, :2 * d].contiguous().view(torch.float16).float() * S8))
        q, k, v = [eff[:, i * d:(i + 1) * d].view(B, T, H, 64).transpose(1, 2) for i in range(3)]
        ref = torch.stack([torch.softmax(q[b, :, row_sel[b]:row_sel[b] + 1] @ k[b].transpose(-1, -2), -1) @ v[b]
                           for b in range(B)]).squeeze(2).reshape(B, d)
        bd = sq_bound(nseg, out_fmt, v.abs().max().item(), ref.abs().max().item())
        worst, bound = max(worst, maxerr(got, ref)), max(bound, bd)
        # the model's full attention kernel on the same planes, rows row_sel[b]
        fout, fldo = attn_out(B * T, d, out_fmt)
        fa = attn_args(op, fout, fldo, B, T, H, nseg, out_fmt)
        _lib.check(lib.pg_attention(C.byref(fa), None))
        torch.cuda.synchronize()
        full = decode_rows(fout, d, out_fmt)[torch.tensor([b * T + r for b, r in enumerate(row_sel)], device="cuda")]
        # the full kernel rounds P to fp16 in the single-fp16 mode (2^-10 * max|out|, test_gpu_kernel_forms.attn_bound)
        worst_full = max(worst_full, maxerr(got, full))
        bound_full = max(bound_full, bd + (2.0 ** -10 * ref.abs().max().item() if nseg == 1 else 3e-5))
    report(f"single-query attention T={T} {MODE_IDS[MODES.index((nseg, out_fmt))]}", worst, bound)
    report(f"single-query vs full attention T={T} {MODE_IDS[MODES.index((nseg, out_fmt))]}", worst_full, bound_full)


# ------------------------------------------------------------------------------------------------ ESM C q/k LayerNorm + rotary
def rotary_tables(T):
    inv = 1.0 / (10000.0 ** (torch.arange(32, dtype=torch.float64) * 2 / 64))
    ang = torch.arange(T, dtype=torch.float64)[:, None] * inv[None, :]
    return torch.cos(ang).float().cuda().contiguous(), torch.sin(ang).float().cuda().contiguous()


def qk_ref(a, g, co, si, T, H, sc):
    """fp64: weight-only LayerNorm over the full row, then rotate-half per 64-wide head at t = row % T, times sc"""
    rows = a.shape[0]
    y = ln64(a, g).view(rows, H, 2, 32)
    t = torch.arange(rows, device="cuda") % T
    c, s = co.double()[t][:, None, :], si.double()[t][:, None, :]
    x1, x2 = y[:, :, 0], y[:, :, 1]
    return torch.stack([x1 * c - x2 * s, x2 * c + x1 * s], 2).reshape(rows, H * 64) * sc


# fp32 statistics over d = 64 H columns and the rotation: 8 * 2^-24 * max|out| for hi + lo (measured 2.1 on an H100 80GB HBM3 at
# 700 W), fp16 rounding, 2^-11 relative, for hi alone (measured 0.82 of it)
QK_BOUND = {0: 2.0 ** -11, 1: 8 * EPS}


@pytest.mark.parametrize("lo", [0, 1], ids=["hi", "hilo"])
@pytest.mark.parametrize("H", [1, 15, 18, 24])
def test_qk_ln_rotary_matches_fp64(H, lo):
    """In place on [q | k] of rows in several windows of T (rows not a multiple of the 8 warps of a block): q and k against fp64 (k
    unscaled, q * 1/8), and the v columns, the lo plane of v and the bytes past the row unchanged bit for bit. A launch with equal q and
    k rows and weights checks that the q scale is exactly 1/8."""
    lib = _lib.load()
    d = H * 64
    worst = bound = 0.0
    for T, nwin in ((5, 3), (37, 2)):
        rows = T * nwin
        gg = gen(H * 10 + lo + T)
        ld = 6 * d + 8 if lo else 3 * d + 8
        x = torch.randn(rows, 3 * d, device="cuda", generator=gg) * 2 + 0.5
        x[:, :2 * d] += torch.linspace(-3, 3, 2 * d, device="cuda")
        buf = torch.randn(rows, ld, device="cuda", generator=gg).half()
        buf[:, :3 * d] = x.half()
        if lo:
            buf[:, 3 * d:6 * d] = (x - x.half().float()).half()
        before = buf.clone()
        qg, kg = torch.randn(d, device="cuda", generator=gg), torch.randn(d, device="cuda", generator=gg)
        co, si = rotary_tables(T)
        _lib.check(lib.pg_qk_ln_rotary(buf.data_ptr(), ld, 3 * d if lo else 0, rows, H, qg.data_ptr(), kg.data_ptr(), co.data_ptr(),
                                       si.data_ptr(), T, None))
        torch.cuda.synchronize()
        assert same_bits(buf[:, 2 * d:3 * d], before[:, 2 * d:3 * d]), "v columns changed"
        assert same_bits(buf[:, (6 if lo else 3) * d:], before[:, (6 if lo else 3) * d:]), "bytes past the row changed"
        if lo:
            assert same_bits(buf[:, 5 * d:6 * d], before[:, 5 * d:6 * d]), "lo plane of v changed"
        a = before[:, :2 * d].double() + (before[:, 3 * d:5 * d].double() if lo else 0)
        got = buf[:, :2 * d].double() + (buf[:, 3 * d:5 * d].double() if lo else 0)
        for half, gam, sc in ((0, qg, 0.125), (1, kg, 1.0)):
            ref = qk_ref(a[:, half * d:(half + 1) * d], gam, co, si, T, H, sc)
            worst = max(worst, maxerr(got[:, half * d:(half + 1) * d], ref))
            bound = max(bound, QK_BOUND[lo] * ref.abs().max().item())
        # q == k rows under equal weights: q comes out exactly k / 8 (the fp16 planes of an exact power-of-two scale, away from subnormals)
        buf2 = before.clone()
        buf2[:, :d] = buf2[:, d:2 * d]
        if lo:
            buf2[:, 3 * d:4 * d] = buf2[:, 4 * d:5 * d]
        _lib.check(lib.pg_qk_ln_rotary(buf2.data_ptr(), ld, 3 * d if lo else 0, rows, H, kg.data_ptr(), kg.data_ptr(), co.data_ptr(),
                                       si.data_ptr(), T, None))
        torch.cuda.synchronize()
        for off in ((0, 3 * d) if lo else (0,)):
            qo, ko = buf2[:, off:off + d].float(), buf2[:, off + d:off + 2 * d].float()
            normal = ko.abs() >= 2.0 ** -10
            assert torch.equal((qo * 8)[normal], ko[normal]), "q is not exactly k / 8"
    report(f"qk LayerNorm + rotary H={H} {'hi/lo' if lo else 'hi'}", worst, bound)


# ------------------------------------------------------------------------------------------------ K5: ESM-family LM head
def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


# fp32 SIMT: three LayerNorms, a d x d dense layer and the vocab dot products of length d, then the lse: c * max(1, max|log p|), where
# the length-d sums make c grow with d (measured 3.0 * 2^-24 at d = 64, 17.4 * 2^-24 at d = 1280 on an H100 80GB HBM3 at 700 W)
MLM_BOUND = 64 * EPS


@pytest.mark.parametrize("vocab", [33, 64])
@pytest.mark.parametrize("d", [64, 320, 480, 1280])
def test_mlm_head_matches_fp64(d, vocab):
    """P rows (1, 63, 64, 65, 200: the dense layer's 64-row tiles) through emb_layer_norm_after -> dense + GELU -> LayerNorm -> tied
    logits + bias -> log_softmax, selected with row_in_seq or taken as they are (all_rows). One output-embedding row is scaled 12x so
    that every row's distribution is peaked and an error in the lse or a LayerNorm term is not averaged away."""
    lib = _lib.load()
    gg = gen(d + vocab)
    rnd = lambda *s, sc=1.0: torch.randn(*s, device="cuda", generator=gg) * sc
    w = dict(lna_g=rnd(d), lna_b=rnd(d), dense_w=rnd(d, d, sc=1.5 / math.sqrt(d)), dense_b=rnd(d), ln_g=rnd(d), ln_b=rnd(d),
             out_w=rnd(vocab, d, sc=1.0 / math.sqrt(d)), out_b=rnd(vocab))
    w["out_w"][7] *= 12.0
    T = 5
    worst = bound = 0.0
    for P in (1, 63, 64, 65, 200):
        for all_rows in (0, 1):
            x = rnd(P if all_rows else P * T, d, sc=2.0) + 1.0
            sel = torch.randint(0, T, (P,), device="cuda", generator=gg, dtype=torch.int32)
            out = torch.full((P + 1, vocab), float("nan"), device="cuda")
            sa, sb = torch.full((P, d), float("nan"), device="cuda"), torch.full((P, d), float("nan"), device="cuda")
            a = _lib.PgMlmHeadArgs(x=x.data_ptr(), d=d, T=T, row_in_seq=None if all_rows else sel.data_ptr(), P=P, all_rows=all_rows,
                                   vocab=vocab, scratch_a=sa.data_ptr(), scratch_b=sb.data_ptr(), out=out.data_ptr(),
                                   **{k: v.data_ptr() for k, v in w.items()})
            _lib.check(lib.pg_mlm_head(C.byref(a), None))
            torch.cuda.synchronize()
            assert torch.isnan(out[P]).all()
            rows = x.double() if all_rows else x.double()[torch.arange(P, device="cuda") * T + sel.long()]
            h = gelu64(ln64(rows, w["lna_g"], w["lna_b"]) @ w["dense_w"].double().T + w["dense_b"].double())
            logits = ln64(h, w["ln_g"], w["ln_b"]) @ w["out_w"].double().T + w["out_b"].double()
            ref = torch.log_softmax(logits, -1)
            worst = max(worst, maxerr(out[:P].double(), ref))
            bound = max(bound, MLM_BOUND * max(1.0, ref.abs().max().item()))
    report(f"MLM head d={d} vocab={vocab}", worst, bound)


# ------------------------------------------------------------------------------------------------ autoregressive head
def ar_ref(x, ids, lens, B, T, vocab, lnf, wte, bias, label_off, ignore_id, fus):
    """fp64 tok_logp [B*T] and fused log-probability rows [B*T, vocab] (NaN where the kernel writes nothing)"""
    y = ln64(x, *lnf) if lnf else x.double()
    logits = y @ wte.double().T
    if bias is not None:
        logits = logits + bias.double()
    lp = torch.log_softmax(logits, -1)
    if fus is not None:
        pr, pr2 = fus["prior_row"].long(), fus.get("prior_row2")
        cols = torch.arange(vocab, device="cuda") >= fus["first_col"]
        mix = (1 - fus["alpha"]) * lp + fus["alpha"] * fus["log_prior"].double()[pr.clamp(min=0)]
        if pr2 is not None:
            pr2 = pr2.long()
            mix = torch.where((pr2 >= 0)[:, None], (1 - fus["beta"]) * mix + fus["beta"] * fus["log_prior2"].double()[pr2.clamp(min=0)], mix)
        fused = torch.where((pr >= 0)[:, None], mix, torch.where((pr == -2)[:, None], (1 - fus["alpha"]) * lp, lp))
        lp = torch.where(cols[None, :], fused, lp)
    tok = torch.zeros(B * T, dtype=torch.float64, device="cuda")
    rows = torch.full((B * T, vocab), float("nan"), dtype=torch.float64, device="cuda")
    idl, lensl = ids.tolist(), lens.tolist()
    for r in range(B * T):
        b, t = divmod(r, T)
        if t + 1 >= lensl[b] or (ignore_id >= 0 and idl[r + 1] == ignore_id):
            continue
        rows[r] = lp[r]
        lab = idl[r + 1] - label_off
        tok[r] = lp[r, lab] if 0 <= lab < vocab else float("nan")
    return tok, rows


AR_CONFIGS = ["tranception", "trancepteve", "progen2", "poet"]
# fp32 LayerNorm, a length-256 dot per logit, the lse and up to two fusion products: c * max(1, max|log p|) (measured 1.7 * 2^-24 on
# an H100 80GB HBM3 at 700 W)
AR_BOUND = 6 * EPS


def seq_sum_check(name, tok, sums, lens, T):
    """out_sum[b] against the fp64 sum of the kernel's own terms t < lens[b] - 1: fewer than 32 terms, one per lane, then five
    butterfly levels of fp32 adds, <= 2.5 ulp of the partial sums: 4 * 2^-24 * sum |terms| (measured ~1 on an H100 80GB HBM3 at
    700 W). A NaN term makes the sum NaN. Reported in units of 2^-24 * sum |terms|."""
    worst = 0.0
    for b, n in enumerate(lens):
        terms = tok[b * T:b * T + max(n - 1, 0)].double()
        ref, got = terms.sum().item(), sums[b].item()
        if math.isnan(ref):
            assert math.isnan(got), (name, b)
            continue
        err = abs(got - ref) if not math.isnan(got) else math.inf
        worst = max(worst, err / (EPS * max(terms.abs().sum().item(), 1e-30)))
    report(f"{name} sequence sums (units of 2^-24 sum|terms|)", worst, 4.0)


@pytest.mark.parametrize("cfg", AR_CONFIGS)
def test_ar_head_matches_fp64(cfg):
    """Each head configuration a decoder launches: Tranception (vocab 25, fusion on every column), TranceptEVE (two-way fusion from
    column 5, prior rows >= 0 / -1 / -2 and second-prior rows >= 0 / -1, the out_logprobs rows), ProGen2 (25 columns from token 5, a
    bias), PoET (vocab 24, target 23 ignored, no LayerNorm). Sequences of length 0, 1, 2 and T; next tokens outside the head's columns
    score NaN; the sequence sums equal the fp64 sums of the terms t < len - 1."""
    lib = _lib.load()
    d, T = 256, 11
    vocab = 24 if cfg == "poet" else 25
    label_off = 5 if cfg == "progen2" else 0
    ignore_id = 23 if cfg == "poet" else -1
    gg = gen(AR_CONFIGS.index(cfg) + 1)
    lens = [0, 1, 2, T, T, 6]
    B = len(lens)
    x = torch.randn(B * T, d, device="cuda", generator=gg) * 2 + 3
    lnf = None if cfg == "poet" else (torch.randn(d, device="cuda", generator=gg), torch.randn(d, device="cuda", generator=gg))
    wte = torch.randn(vocab, d, device="cuda", generator=gg) / math.sqrt(d) * 2
    bias = torch.randn(vocab, device="cuda", generator=gg) if cfg == "progen2" else None
    ids = torch.randint(label_off, label_off + vocab, (B * T,), device="cuda", generator=gg, dtype=torch.int32)
    # sequence 4 (len T): next tokens outside the head's columns; sequence 3: token 5 (TranceptEVE's first fused column) as target
    ids[4 * T + 3], ids[4 * T + 6] = label_off + vocab, label_off - 1
    ids[3 * T + 1:3 * T + 6] = 5
    if cfg == "poet":
        ids[3 * T + 7] = ids[5 * T + 2] = ids[4 * T + 8] = 23  # ignored, also in the sequence with the NaN targets
    ids = ids.contiguous()
    fus, f = None, None
    if cfg in ("tranception", "trancepteve"):
        n_prior = 9
        lp1 = torch.log_softmax(torch.randn(n_prior, vocab, device="cuda", generator=gg) * 3, -1)
        pr = torch.randint(0, n_prior, (B * T,), device="cuda", generator=gg, dtype=torch.int32)
        pr[::4] = -1
        fus = dict(log_prior=lp1, prior_row=pr, alpha=0.6, first_col=0)
        if cfg == "trancepteve":
            pr[1::4] = -2
            lp2 = torch.log_softmax(torch.randn(n_prior, vocab, device="cuda", generator=gg) * 3, -1)
            pr2 = torch.randint(0, n_prior, (B * T,), device="cuda", generator=gg, dtype=torch.int32)
            pr2[::3] = -1
            fus.update(log_prior2=lp2, prior_row2=pr2, beta=0.3, first_col=5)
        out_lp = torch.full((B * T, vocab), float("nan"), device="cuda")
        f = _lib.PgArFusion(log_prior=lp1.data_ptr(), prior_row=pr.data_ptr(), alpha=fus["alpha"], first_col=fus["first_col"],
                            out_logprobs=out_lp.data_ptr())
        if cfg == "trancepteve":
            f.log_prior2, f.prior_row2, f.beta = lp2.data_ptr(), pr2.data_ptr(), fus["beta"]
    tok = torch.full((B * T,), float("nan"), device="cuda")
    sums = torch.full((B + 1,), float("nan"), device="cuda")
    lens_t = i32(lens)
    a = _lib.PgArHeadArgs(x=x.data_ptr(), d=d, B=B, T=T, vocab=vocab, ids=ids.data_ptr(), lens=lens_t.data_ptr(),
                          lnf_g=ptr(lnf[0]) if lnf else None, lnf_b=ptr(lnf[1]) if lnf else None, wte=wte.data_ptr(), bias=ptr(bias),
                          label_off=label_off, ignore_id=ignore_id, tok_logp=tok.data_ptr(), out_sum=sums.data_ptr())
    _lib.check(lib.pg_ar_head(C.byref(a), C.byref(f) if f is not None else None, None))
    torch.cuda.synchronize()
    assert torch.isnan(sums[B])
    ref_tok, ref_rows = ar_ref(x, ids, lens_t, B, T, vocab, lnf, wte, bias, label_off, ignore_id, fus)
    got = tok.double()
    assert torch.equal(torch.isnan(got), torch.isnan(ref_tok)), "NaN targets"
    assert torch.isnan(ref_tok).sum().item() == 2
    zero = ref_tok == 0  # beyond the length, and ignored targets: exactly 0
    assert (got[zero] == 0).all() and not (got[~zero] == 0).any()
    fin = ~torch.isnan(ref_tok)
    bound = AR_BOUND * max(1.0, ref_tok[fin].abs().max().item())
    worst = maxerr(got[fin], ref_tok[fin])
    if fus is not None:
        written = ~torch.isnan(ref_rows[:, 0])
        assert torch.isnan(out_lp[~written]).all(), "out_logprobs rows written beyond the length"
        worst = max(worst, maxerr(out_lp.double()[written], ref_rows[written]))
    report(f"AR head {cfg}", worst, bound)
    seq_sum_check(f"AR head {cfg}", tok, sums, lens, T)


# ------------------------------------------------------------------------------------------------ LM-head combine (after epi 7)
# the (max, sum) pairs are fp32 roundings of fp64 values (2^-24 relative each), merged with expf / logf over `tiles` pairs: a few ulp
# of max(|lse|, 1) plus 2^-24 per merge level; the in-place rows add one rounding of |logit - lse|. Measured 0.27 of this bound
# (the in-place rows of a tile 150 below the row max) on an H100 80GB HBM3 at 700 W.
def combine_bound(lse_max, lp_max):
    return 16 * EPS * max(1.0, lse_max) + 2 * EPS * lp_max


@pytest.mark.parametrize("tiles", [1, 2, 31, 32, 33, 393])
def test_lm_combine_matches_fp64(tiles):
    """Partials built in fp64 from known fp32 logits, one tile per row 150 below the row's max (its exp underflows) and one 3 above the
    rest; tok_logp = target logit - lse, NaN for labels -1 and vocab, 0 beyond the length; out_logprobs rows turned into logit - lse in
    place, the other rows left bit for bit; the sequence sums against the fp64 sums of the terms. 393 tiles are ProtGPT2's ceil(50 257 / 128)."""
    lib = _lib.load()
    vocab = {1: 100, 2: 200, 31: 31 * 128 - 5, 32: 32 * 128, 33: 33 * 128 - 100, 393: 50257}[tiles]
    T, lens = 6, [0, 1, 3, 6, 6]
    B = len(lens)
    rows = B * T
    gg = gen(tiles)
    L = torch.randn(rows, vocab, device="cuda", generator=gg) * 2
    col_tile = torch.arange(vocab, device="cuda") // 128
    for r in range(rows):
        hot, cold = (r * 7) % tiles, (r * 3 + 1) % tiles
        L[r, col_tile == hot] += 3.0
        if cold != hot:
            L[r, col_tile == cold] -= 150.0
    L64 = L.double()
    part = torch.zeros(rows, tiles, 2, dtype=torch.float64, device="cuda")
    for k in range(tiles):
        blk = L64[:, k * 128:(k + 1) * 128]
        m = blk.max(1).values
        part[:, k, 0], part[:, k, 1] = m, torch.exp(blk - m[:, None]).sum(1)
    part = part.float().contiguous()
    ids = torch.randint(0, vocab, (rows,), device="cuda", generator=gg, dtype=torch.int32)
    ids[3 * T + 2], ids[4 * T + 4] = -1, vocab
    tgt = L[torch.arange(rows, device="cuda"), ids.long().clamp(0, vocab - 1).roll(-1)].contiguous()
    logits = L.clone()
    tok = torch.full((rows,), float("nan"), device="cuda")
    sums = torch.full((B + 1,), float("nan"), device="cuda")
    _lib.check(lib.pg_lm_combine(part.data_ptr(), tiles, tgt.data_ptr(), ids.data_ptr(), i32(lens).data_ptr(), B, T, vocab,
                                 logits.data_ptr(), tok.data_ptr(), sums.data_ptr(), None))
    torch.cuda.synchronize()
    assert torch.isnan(sums[B])
    lse = torch.logsumexp(L64, 1)
    live = torch.tensor([(r % T) + 1 < lens[r // T] for r in range(rows)], device="cuda")
    idl = ids.tolist()
    ref_tok = torch.zeros(rows, dtype=torch.float64, device="cuda")
    for r in range(rows):
        if live[r]:
            lab = idl[r + 1]
            ref_tok[r] = tgt[r].double() - lse[r] if 0 <= lab < vocab else float("nan")
    got = tok.double()
    assert torch.equal(torch.isnan(got), torch.isnan(ref_tok)) and torch.isnan(ref_tok).sum().item() == 2
    assert (got[~live] == 0).all()
    fin = live & ~torch.isnan(ref_tok)
    ref_rows = L64[live] - lse[live][:, None]
    worst = max(maxerr(got[fin], ref_tok[fin]), maxerr(logits.double()[live], ref_rows))
    assert same_bits(logits[~live], L[~live]), "rows beyond the length changed"
    bound = combine_bound(lse.abs().max().item(), ref_rows.abs().max().item())
    report(f"LM combine tiles={tiles}", worst, bound)
    seq_sum_check(f"LM combine tiles={tiles}", tok, sums, lens, T)


# ------------------------------------------------------------------------------------------------ argument checks
def test_row_entry_points_refuse_bad_arguments():
    """Bad sizes and missing buffers return PG_ERR_ARG (unsupported forms PG_ERR_UNSUPPORTED) and launch nothing."""
    lib = _lib.load()
    f32 = torch.zeros(64, 64, device="cuda")
    i = i32([0, 1, 2, 3])
    sentinel = torch.full((64, 64), float("nan"), device="cuda")
    # single-query attention
    qkv = torch.zeros(8, 3 * 64, device="cuda", dtype=torch.float16)
    out = sentinel.view(torch.float16)
    for field, value, code in (("T", 0, PG_ERR_ARG), ("heads", 0, PG_ERR_ARG), ("nseg", 2, PG_ERR_ARG), ("ld", 100, PG_ERR_ARG),
                               ("causal", 1, PG_ERR_UNSUPPORTED), ("impl", 1, PG_ERR_UNSUPPORTED), ("ldo", 32, PG_ERR_ARG),
                               ("out_fmt", 2, PG_ERR_ARG)):
        a = _lib.PgAttnArgs(qkv=qkv.data_ptr(), ld=3 * 64, out=out.data_ptr(), ldo=64, B=2, T=4, heads=1, nseg=1)
        setattr(a, field, value)
        assert lib.pg_attention_rows(C.byref(a), i.data_ptr(), None) == code, field
    a = _lib.PgAttnArgs(qkv=qkv.data_ptr(), ld=3 * 64, out=out.data_ptr(), ldo=64, B=2, T=4, heads=1, nseg=3)  # x3 without a lo plane
    assert lib.pg_attention_rows(C.byref(a), i.data_ptr(), None) == PG_ERR_ARG
    a.nseg = 1
    assert lib.pg_attention_rows(C.byref(a), None, None) == PG_ERR_ARG
    # q/k LayerNorm + rotary
    p = f32.data_ptr()
    assert lib.pg_qk_ln_rotary(qkv.data_ptr(), 3 * 64, 0, 8, 25, p, p, p, p, 4, None) == PG_ERR_ARG     # heads > 24
    assert lib.pg_qk_ln_rotary(qkv.data_ptr(), 3 * 64, 0, 8, 1, p, p, p, p, 0, None) == PG_ERR_ARG      # T = 0
    assert lib.pg_qk_ln_rotary(qkv.data_ptr(), 3 * 64, 0, 8, 1, None, p, p, p, 4, None) == PG_ERR_ARG   # no q weight
    assert lib.pg_qk_ln_rotary(qkv.data_ptr(), 100, 0, 8, 1, p, p, p, p, 4, None) == PG_ERR_ARG         # row narrower than [q | k]
    assert lib.pg_qk_ln_rotary(qkv.data_ptr(), 3 * 64, 64, 8, 1, p, p, p, p, 4, None) == PG_ERR_ARG     # lo plane inside [q | k]
    # embedding
    e = _lib.PgEsmEmbedArgs(tokens=i.data_ptr(), n_tokens=4, P=2, T=0, d=64, embed=p, x=sentinel.data_ptr())
    assert lib.pg_esm_embed(C.byref(e), None) == PG_ERR_ARG
    e.T, e.n_tokens = 4, 0
    assert lib.pg_esm_embed(C.byref(e), None) == PG_ERR_ARG
    e.n_tokens, e.lnb_gamma = 4, p  # LayerNorm weight without its bias
    assert lib.pg_esm_embed(C.byref(e), None) == PG_ERR_ARG
    # MLM head
    h = _lib.PgMlmHeadArgs(x=p, d=64, T=4, P=2, all_rows=0, vocab=33, scratch_a=p, scratch_b=p, out=sentinel.data_ptr(),
                           **{k: p for k in ("lna_g", "lna_b", "dense_w", "dense_b", "ln_g", "ln_b", "out_w", "out_b")})
    assert lib.pg_mlm_head(C.byref(h), None) == PG_ERR_ARG  # row_in_seq missing
    h.all_rows, h.vocab = 1, 0
    assert lib.pg_mlm_head(C.byref(h), None) == PG_ERR_ARG
    h.vocab, h.d = 33, 12288
    assert lib.pg_mlm_head(C.byref(h), None) == PG_ERR_ARG  # row + logits beyond 48 KB of shared memory
    # AR head
    ar = _lib.PgArHeadArgs(x=p, d=64, B=1, T=4, vocab=25, ids=i.data_ptr(), lens=i.data_ptr(), lnf_g=p, lnf_b=None, wte=p,
                           ignore_id=-1, tok_logp=sentinel.data_ptr(), out_sum=sentinel.data_ptr())
    assert lib.pg_ar_head(C.byref(ar), None, None) == PG_ERR_ARG  # lnf_g without lnf_b
    ar.lnf_b = p
    bad = _lib.PgArFusion(log_prior=p, prior_row=None)
    assert lib.pg_ar_head(C.byref(ar), C.byref(bad), None) == PG_ERR_ARG
    bad = _lib.PgArFusion(log_prior=p, prior_row=i.data_ptr(), first_col=26)
    assert lib.pg_ar_head(C.byref(ar), C.byref(bad), None) == PG_ERR_ARG
    ar.T = 0
    assert lib.pg_ar_head(C.byref(ar), None, None) == PG_ERR_ARG
    # combine
    s = sentinel.data_ptr()
    assert lib.pg_lm_combine(p, 0, p, i.data_ptr(), i.data_ptr(), 1, 4, 100, None, s, s, None) == PG_ERR_ARG
    assert lib.pg_lm_combine(p, 1, p, i.data_ptr(), i.data_ptr(), -1, 4, 100, None, s, s, None) == PG_ERR_ARG
    assert lib.pg_lm_combine(p, 1, p, None, i.data_ptr(), 1, 4, 100, None, s, s, None) == PG_ERR_ARG
    torch.cuda.synchronize()
    assert torch.isnan(sentinel).all()
