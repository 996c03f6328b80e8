"""GPU (-m gpu): the attention (K4) and GEMM (K3) forms that only some model stacks launch, kernel by kernel through pg_attention_form /
pg_gemm_form, against fp64 evaluations of the operand planes the kernels read and, where a form only reorders or skips work, for
bit-identity with the plain form that computes the same thing.

Inputs are built so that a wrong mask moves the result by O(1): keys that must stay hidden (padding rows, other segments, the next
sequence) get scores far above the visible ones. Every test prints its measured error next to its bound."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from proteingym_b200 import _lib
from test_gpu_parity import dq8, hilo, pack_a_f8, unpack_f8

pytestmark = pytest.mark.gpu
S_OUT = 4.0     # e4m3 scale of out_fmt 2 outputs
S_A = 4.0       # e4m3 scale of nseg-2 `a` operands
MODES = [(1, 0), (3, 1), (3, 2)]  # attention (nseg, out_fmt): single fp16; hi/lo x3 into fp16 hi/lo; hi/lo x3 into e4m3 planes
MODE_IDS = ["nseg1", "nseg3-fmt1", "nseg3-fmt2"]
KCHUNK_DEFAULT, CTA2_DEFAULT, PREFETCH_DEFAULT = 1280, 1, 0  # pg_set_tuning defaults (include/pgscore.h)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def report(name, err, bound):
    print(f"\n[kernel forms] {name}: max|err| = {err:.3e} (bound {bound:.3e})")
    assert err < bound, (name, err, bound)


# ------------------------------------------------------------------------------------------------ attention (K4)
def pack_qkv(x, nseg):
    """fp32 [rows, 3d] -> (fp16 operand rows, the fp64 values the kernel reads: hi, or hi + lo)."""
    d3 = x.shape[1]
    if nseg == 3:
        t = hilo(x)
        return t, t[:, :d3].double() + t[:, d3:].double()
    t = x.half().contiguous()
    return t, t.double()


def run_attn(op, B, T, H, nseg, out_fmt, causal=1, hd=64, slopes=None, **form):
    """One pg_attention_form launch over B sequences of T rows of `op` -> the raw output buffer (unwritten bytes stay NaN)."""
    lib = _lib.load()
    d = H * hd
    rows = B * T
    if out_fmt == 2:
        out = torch.full((rows, 4 * d), 0xFF, device="cuda", dtype=torch.uint8)
    else:
        out = torch.full((rows, d * (2 if out_fmt else 1)), float("nan"), device="cuda", dtype=torch.float16)
    a = _lib.PgAttnArgs()
    a.qkv, a.ld, a.lo_off = op.data_ptr(), op.shape[1], (3 * d if nseg == 3 else 0)
    a.out, a.ldo, a.out_lo_off = out.data_ptr(), (2 * d if out_fmt else d), (d if out_fmt else 0)
    a.B, a.T, a.heads, a.nseg, a.causal, a.impl = B, T, H, nseg, causal, 0
    a.alibi_slopes = slopes.data_ptr() if slopes is not None else None
    a.out_fmt, a.out_scale = out_fmt, (S_OUT if out_fmt == 2 else 0.0)
    f = _lib.PgAttnForm(head_dim=hd)
    for k, v in form.items():
        setattr(f, k, v)
    _lib.check(lib.pg_attention_form(C.byref(a), C.byref(f), None))
    torch.cuda.synchronize()
    return out


def decode(out, d, out_fmt):
    """Output rows -> fp64 values (hi + lo, or hi + lo8 / (2^11 s))."""
    if out_fmt == 0:
        return out[:, :d].double()
    if out_fmt == 1:
        return out[:, :d].double() + out[:, d:].double()
    hi, lo8, _ = unpack_f8(out, d, S_OUT)
    return hi + lo8


# fp16 hi/lo x3 attention error (into fp16 hi / lo planes) per form: about 3x the largest error measured over the form's cases on an
# H100 80GB HBM3 (700 W): shared prefix 1.3e-5, memory form 7.4e-6 (at P = 1; 1.4e-7 at P = 6145), segment-causal 9.1e-6,
# next-sequence rows 5.0e-6, memory form over a 24 576 / 24 640-row record 7.7e-8
X3_BOUND = {"prefix": 4e-5, "memory": 2.5e-5, "segment": 3e-5, "tail": 1.5e-5, "long": 3e-7}


def attn_bound(nseg, out_fmt, vmax, form):
    """Single fp16: P and the output are rounded to fp16 (2^-11 relative each), at most 2^-10 * max|out| (measured <= 1.3e-3 at
    max|out| ~ 3.5, 2.7x under). x3 scheme: the form's measured fp32 softmax / accumulation error; e4m3 planes add the low part
    carried at 4 bits instead of 11, 2^-16 * max|out| (measured 3.5e-5 at ~3.5)."""
    if nseg == 1:
        return 2.0 ** -10 * vmax
    return X3_BOUND[form] + (2.0 ** -16 * vmax if out_fmt == 2 else 0.0)


def heads_of(x, H, hd):
    """[rows, H * hd] -> [H, rows, hd]"""
    return x.view(x.shape[0], H, hd).transpose(0, 1)


def attend(q, k, v, vis, bias=None):
    """fp64 softmax(q k^T + bias, masked to `vis`) v; q [H, Tq, w], k / v [H, Tk, w], vis [Tq, Tk] bool."""
    s = q @ k.transpose(-1, -2)
    if bias is not None:
        s = s + bias
    s = s.masked_fill(~vis, float("-inf"))
    return torch.softmax(s, -1) @ v


def angle_qkv(rows, group, H, hd, g, noise=0.25):
    """q / k / v rows whose q . k is -10 within a group and up to +7.4 between groups: group i sits at angle i * 137.5 degrees in
    columns 0-1 of every head, q pointing away from its own group's keys. A key leaking in from another group takes nearly all the
    weight. group: [rows] int64 (device)."""
    th = group.double() * (2 * math.pi * 0.381966011250105)
    x = torch.randn(rows, 3, H, hd, device="cuda", generator=g) * noise
    r = math.sqrt(10.0)
    x[:, 0, :, 0] = (-r * torch.cos(th))[:, None].float()
    x[:, 0, :, 1] = (-r * torch.sin(th))[:, None].float()
    x[:, 1, :, 0] = (r * torch.cos(th))[:, None].float()
    x[:, 1, :, 1] = (r * torch.sin(th))[:, None].float()
    x[:, 2] = torch.randn(rows, H, hd, device="cuda", generator=g)
    return x.reshape(rows, 3 * H * hd)


def slot_pad(x, H, w, hd):
    """[rows, 3 * H * w] -> [rows, 3 * H * hd] with columns w .. hd of every head slot zero (ProGen2's 80- and 96-wide heads)."""
    if w == hd:
        return x
    y = torch.zeros(x.shape[0], 3, H, hd, device=x.device, dtype=x.dtype)
    y[..., :w] = x.view(x.shape[0], 3, H, w)
    return y.reshape(x.shape[0], 3 * H * hd)


@pytest.mark.parametrize("P", [128, 256])
@pytest.mark.parametrize("w", [64, 80, 96])
@pytest.mark.parametrize("nseg,out_fmt", MODES, ids=MODE_IDS)
def test_shared_prefix_matches_fp64_and_full_launch(nseg, out_fmt, w, P):
    """Causal attention over a shared prefix of P rows (K / V in `prefix`) + T own rows, with and without ALiBi at the absolute key
    index; 64-wide slots, or 80 / 96-wide heads in 128-wide slots. The own rows must equal, bit for bit, rows [P, P + T) of a plain
    causal launch over the concatenated sequences: both visit the same key blocks in the same order."""
    hd = 64 if w == 64 else 128
    worst, bound = 0.0, 0.0
    for H in (1, 4):
        d = H * hd
        g = torch.Generator(device="cuda").manual_seed(P + w + H)
        pre = slot_pad(torch.randn(P, 3 * H * w, device="cuda", generator=g), H, w, hd)
        pre[:, :d] *= 0.3
        pre_op, pre_eff = pack_qkv(pre, nseg)
        for B in (1, 3):
            for T in (1, 63, 64, 65, 129):
                own = slot_pad(torch.randn(B * T, 3 * H * w, device="cuda", generator=g), H, w, hd)
                own[:, :d] *= 0.3
                own_op, own_eff = pack_qkv(own, nseg)
                full_op = torch.cat([torch.cat([pre_op, own_op[b * T:(b + 1) * T]]) for b in range(B)]).contiguous()
                for alibi in (0, 1):
                    slopes = torch.tensor([2.0 ** -(i + 3) for i in range(H)], device="cuda") if alibi else None
                    out = run_attn(own_op, B, T, H, nseg, out_fmt, 1, hd, slopes, prefix=pre_op.data_ptr(), prefix_len=P)
                    ref_full = run_attn(full_op, B, P + T, H, nseg, out_fmt, 1, hd, slopes)
                    sel = torch.cat([torch.arange(b * (P + T) + P, (b + 1) * (P + T), device="cuda") for b in range(B)])
                    assert same_bits(out, ref_full[sel]), (H, B, T, alibi)
                    got = decode(out, d, out_fmt)
                    if w < hd:  # the zero columns of each slot stay zero
                        assert not heads_of(got, H, hd)[..., w:].any()
                    kv = [torch.cat([pre_eff, own_eff[b * T:(b + 1) * T]]) for b in range(B)]
                    j = torch.arange(P + T, device="cuda")
                    vis = j[None, :] <= (P + torch.arange(T, device="cuda"))[:, None]
                    for b in range(B):
                        bias = slopes.double()[:, None, None] * j.double()[None, None, :] if alibi else None
                        ref = attend(heads_of(own_eff[b * T:(b + 1) * T, :d], H, hd), heads_of(kv[b][:, d:2 * d], H, hd),
                                     heads_of(kv[b][:, 2 * d:], H, hd), vis, bias)
                        r = ref.transpose(0, 1).reshape(T, d)
                        worst = max(worst, (got[b * T:(b + 1) * T] - r).abs().max().item())
                        bound = max(bound, attn_bound(nseg, out_fmt, r.abs().max().item(), "prefix"))
    report(f"shared prefix P={P} width {w}/{hd} {MODE_IDS[MODES.index((nseg, out_fmt))]}", worst, bound)


def unit_dirs(H, g):
    u = torch.randn(H, 64, device="cuda", generator=g)
    return u / u.norm(dim=1, keepdim=True)


def record_qkv(rows, u, g):
    """Rows for the memory form: every key near the direction u[h] of its head and every q near -3 u[h], so that every real score is
    about -10.5 (<= -8). A padding row of the record is zero-filled by TMA and scores exactly 0, so one leaked row takes most of the
    weight."""
    H = u.shape[0]
    x = torch.randn(rows, 3, H, 64, device="cuda", generator=g)
    x[:, 0] = -3.0 * u + 0.1 * x[:, 0]
    x[:, 1] = 3.5 * u + 0.1 * x[:, 1]
    return x.reshape(rows, 3 * H * 64)


def memory_ref(mem_eff, own_eff, B, T, H, P):
    d = H * 64
    j = torch.arange(P + T, device="cuda")
    vis = j[None, :] < P + 1 + torch.arange(T, device="cuda")[:, None]
    refs, smax = [], -float("inf")
    for b in range(B):
        o = own_eff[b * T:(b + 1) * T]
        kv = torch.cat([mem_eff, o])
        q, k = heads_of(o[:, :d], H, 64), heads_of(kv[:, d:2 * d], H, 64)
        smax = max(smax, (q @ k.transpose(-1, -2)).masked_fill(~vis, -1e9).max().item())
        refs.append(attend(q, k, heads_of(kv[:, 2 * d:], H, 64), vis).transpose(0, 1).reshape(T, d))
    return torch.cat(refs), smax


@pytest.mark.parametrize("P", [1, 63, 64, 65, 127, 129, 6145])
@pytest.mark.parametrize("nseg,out_fmt", MODES, ids=MODE_IDS)
def test_memory_form_matches_fp64_and_is_batch_independent(nseg, out_fmt, P):
    """PoET's variant rows against the context record: P record rows of any length, all visible, the tail of the last key block
    masked; work items in head-major order. B = 5 must equal, bit for bit, launches of B = 2 and B = 3 on the same rows."""
    worst, bound = 0.0, 0.0
    for H in (1, 16):
        d = H * 64
        g = torch.Generator(device="cuda").manual_seed(P * 7 + H)
        u = unit_dirs(H, g)
        mem_op, mem_eff = pack_qkv(record_qkv(P, u, g), nseg)
        for B in (1, 5):
            for T in (1, 2, 63, 64, 65, 129):
                own_op, own_eff = pack_qkv(record_qkv(B * T, u, g), nseg)
                form = dict(prefix=mem_op.data_ptr(), prefix_len=P, prefix_mem=1)
                out = run_attn(own_op, B, T, H, nseg, out_fmt, **form)
                ref, smax = memory_ref(mem_eff, own_eff, B, T, H, P)
                assert smax <= -8.0, smax  # the inputs do what they are built for
                got = decode(out, d, out_fmt)
                worst = max(worst, (got - ref).abs().max().item())
                bound = max(bound, attn_bound(nseg, out_fmt, ref.abs().max().item(), "memory"))
                if B == 5:
                    lo = run_attn(own_op[:2 * T].contiguous(), 2, T, H, nseg, out_fmt, **form)
                    hi = run_attn(own_op[2 * T:].contiguous(), 3, T, H, nseg, out_fmt, **form)
                    assert same_bits(out, torch.cat([lo, hi])), (H, T)
    report(f"memory form P={P} {MODE_IDS[MODES.index((nseg, out_fmt))]}", worst, bound)


@pytest.mark.parametrize("nseg,out_fmt", MODES, ids=MODE_IDS)
def test_memory_form_long_record(nseg, out_fmt):
    """A PoET-sized record (P = 24 640 rows) against fp64. At P = 24 576, a multiple of 128, every record row is visible in both forms,
    so the shared-prefix form computes the same attention on the same data: both errors are printed, to show what adding each key
    block's P V in round-to-nearest fp32 (memory form) buys over the tensor core's own accumulation. Only the memory form is held to
    a bound."""
    B, T, H = 2, 65, 2
    d = H * 64
    g = torch.Generator(device="cuda").manual_seed(24640)
    u = unit_dirs(H, g)
    mem_op, mem_eff = pack_qkv(record_qkv(24640, u, g), nseg)
    own_op, own_eff = pack_qkv(record_qkv(B * T, u, g), nseg)
    errs = {}
    for P, mem in ((24640, 1), (24576, 1), (24576, 0)):
        out = run_attn(own_op, B, T, H, nseg, out_fmt, prefix=mem_op.data_ptr(), prefix_len=P, prefix_mem=mem)
        ref, smax = memory_ref(mem_eff[:P], own_eff, B, T, H, P)
        assert smax <= -8.0, smax
        errs[(P, mem)] = (decode(out, d, out_fmt) - ref).abs().max().item()
        if mem:
            bound = attn_bound(nseg, out_fmt, ref.abs().max().item(), "long")
    print(f"\n[kernel forms] long record {MODE_IDS[MODES.index((nseg, out_fmt))]}: P=24640 memory form {errs[(24640, 1)]:.3e}; "
          f"P=24576 memory form {errs[(24576, 1)]:.3e}, shared-prefix form {errs[(24576, 0)]:.3e}")
    report(f"long record P=24640 {MODE_IDS[MODES.index((nseg, out_fmt))]}", max(errs[(24640, 1)], errs[(24576, 1)]), bound)


def poet_lengths():
    rng = np.random.RandomState(0)
    lens, rest = [], 24640
    while rest > 700:
        lens.append(int(rng.randint(3, min(700, rest - 3) + 1)))
        rest -= lens[-1]
    return lens + [rest]


SEGMENTS = {
    "ones200": [1] * 200,
    "63-1-65-300": [63, 1, 65, 300],
    "tile20": [5, 1, 3, 2, 4, 1, 6, 2, 3, 3, 1, 4, 2, 5, 3, 2, 4, 6, 2, 5],
    "one6145": [6145],
    "poet24640": poet_lengths(),
}


@pytest.mark.parametrize("segs", list(SEGMENTS))
@pytest.mark.parametrize("nseg,out_fmt", MODES, ids=MODE_IDS)
def test_segment_causal_matches_fp64(nseg, out_fmt, segs):
    """PoET's context self-attention: one packed sequence of segments, row t seeing keys seg_start[t] .. t; key blocks before the
    query tile's first segment are skipped. Keys of other segments score up to +7.4 against -10 inside the segment."""
    lens = SEGMENTS[segs]
    T, H = sum(lens), 2
    d = H * 64
    group = torch.cat([torch.full((n,), i, dtype=torch.int64) for i, n in enumerate(lens)]).cuda()
    starts = torch.tensor(np.repeat(np.cumsum([0] + lens[:-1]), lens), dtype=torch.int32, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(T)
    op, eff = pack_qkv(angle_qkv(T, group, H, 64, g), nseg)
    out = run_attn(op, 1, T, H, nseg, out_fmt, seg_start=starts.data_ptr())
    got = decode(out, d, out_fmt)
    ref = torch.empty(T, d, device="cuda", dtype=torch.float64)
    for s0, n in zip(np.cumsum([0] + lens[:-1]).tolist(), lens):
        x = eff[s0:s0 + n]
        vis = torch.ones(n, n, device="cuda", dtype=torch.bool).tril()
        ref[s0:s0 + n] = attend(heads_of(x[:, :d], H, 64), heads_of(x[:, d:2 * d], H, 64), heads_of(x[:, 2 * d:], H, 64),
                                vis).transpose(0, 1).reshape(n, d)
    if segs == "ones200":  # every row sees only itself: the output is its own v, up to the rounding of the output
        if nseg == 1:
            assert same_bits(out[:, :d], op[:, 2 * d:3 * d])
    if len(lens) == 1:  # one segment is plain causal attention
        assert same_bits(out, run_attn(op, 1, T, H, nseg, out_fmt))
    report(f"segment-causal {segs} {MODE_IDS[MODES.index((nseg, out_fmt))]}", (got - ref).abs().max().item(),
           attn_bound(nseg, out_fmt, ref.abs().max().item(), "segment"))


@pytest.mark.parametrize("n,L", [(4, 192), (3, 64), (2, 1024)])
@pytest.mark.parametrize("nseg,out_fmt", MODES, ids=MODE_IDS)
def test_segment_causal_equal_segments_match_batched_launch(nseg, out_fmt, n, L):
    """n equal segments of a multiple of 64 rows = a plain causal launch over n sequences, bit for bit."""
    H = 2
    group = torch.arange(n * L, device="cuda") // L
    starts = (group * L).to(torch.int32)
    g = torch.Generator(device="cuda").manual_seed(n * L)
    op, _ = pack_qkv(angle_qkv(n * L, group, H, 64, g), nseg)
    out = run_attn(op, 1, n * L, H, nseg, out_fmt, seg_start=starts.data_ptr())
    assert same_bits(out, run_attn(op, n, L, H, nseg, out_fmt))


@pytest.mark.parametrize("C", [1, 3, 130])
@pytest.mark.parametrize("R", [1, 63, 64, 65, 1024])
@pytest.mark.parametrize("nseg,out_fmt", MODES, ids=MODE_IDS)
def test_column_form_is_permuted_plain_launch(nseg, out_fmt, R, C):
    """The MSA Transformer's column attention: sequence (b, c) of R rows writes its row r to output row (b, r, c). The output must be,
    bit for bit, the plain launch over the same B * C sequences with its rows permuted."""
    nb, H = (1 if R * C > 100000 else 2), 2
    d = H * 64
    g = torch.Generator(device="cuda").manual_seed(R * C)
    x = torch.randn(nb * C * R, 3 * d, device="cuda", generator=g)
    x[:, :d] *= 0.3
    op, _ = pack_qkv(x, nseg)
    out = run_attn(op, nb * C, R, H, nseg, out_fmt, causal=0, perm_C=C)
    plain = run_attn(op, nb * C, R, H, nseg, out_fmt, causal=0)
    perm = plain.view(nb, C, R, -1).transpose(1, 2).reshape(nb * R * C, -1)
    assert same_bits(out, perm)


@pytest.mark.parametrize("T", [63, 65, 129])
@pytest.mark.parametrize("nseg,out_fmt", MODES, ids=MODE_IDS)
def test_next_sequence_rows_stay_hidden(nseg, out_fmt, T):
    """B = 3 sequences whose last key block runs into the next sequence's rows, which score up to +7.4 against -10 inside the
    sequence: the `key >= T` mask is all that hides them. Plain (bidirectional and causal), column, shared-prefix and memory forms."""
    B, H = 3, 2
    d = H * 64
    group = torch.arange(B * T, device="cuda") // T
    g = torch.Generator(device="cuda").manual_seed(T)
    op, eff = pack_qkv(angle_qkv(B * T, group, H, 64, g), nseg)
    # a prefix from the same construction as sequence 0: its keys, too, are visible to every row of every sequence
    pre_op, pre_eff = pack_qkv(angle_qkv(128, torch.full((128,), 5, device="cuda"), H, 64, g), nseg)
    worst, bound = 0.0, 0.0
    for form in ("bidirectional", "causal", "column", "prefix", "memory"):
        kw = {}
        P = 0
        if form == "column":
            kw = dict(perm_C=B)
        if form in ("prefix", "memory"):
            P = 128 if form == "prefix" else 65
            kw = dict(prefix=pre_op.data_ptr(), prefix_len=P, prefix_mem=int(form == "memory"))
        causal = int(form not in ("bidirectional", "column"))
        out = run_attn(op, B, T, H, nseg, out_fmt, causal=causal, **kw)
        got = decode(out, d, out_fmt)
        if form == "column":
            got = got.view(T, B, d).transpose(0, 1).reshape(B * T, d)
        for b in range(B):
            x = torch.cat([pre_eff[:P], eff[b * T:(b + 1) * T]])
            n = P + T
            vis = torch.ones(T, n, device="cuda", dtype=torch.bool)
            if causal:
                vis = torch.arange(n, device="cuda")[None, :] <= P + torch.arange(T, device="cuda")[:, None]
            r = attend(heads_of(x[P:, :d], H, 64), heads_of(x[:, d:2 * d], H, 64), heads_of(x[:, 2 * d:], H, 64), vis)
            r = r.transpose(0, 1).reshape(T, d)
            worst = max(worst, (got[b * T:(b + 1) * T] - r).abs().max().item())
            bound = max(bound, attn_bound(nseg, out_fmt, r.abs().max().item(), "tail"))
    report(f"next-sequence rows T={T} {MODE_IDS[MODES.index((nseg, out_fmt))]}", worst, bound)


# ------------------------------------------------------------------------------------------------ GEMM (K3)
class GemmOp:
    """Operands of one GEMM in the format of `nseg` and the fp64 product of the planes the kernel reads (`ref`, without bias)."""

    def __init__(self, M, N, K, nseg, seed, a_gain=1.0):
        lib = _lib.load()
        g = torch.Generator(device="cuda").manual_seed(seed)
        A = torch.randn(M, K, device="cuda", generator=g) * a_gain
        W = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
        self.M, self.N, self.K, self.nseg = M, N, K, nseg
        self.w_inv = None
        self.bias = torch.randn(N, device="cuda", generator=g)
        if nseg == 1:
            self.a, self.w = A.half().contiguous(), W.half().contiguous()
            self.ref = self.a.double() @ self.w.double().T
        elif nseg == 3:
            self.a, self.w = hilo(A), hilo(W)
            ah, wh = self.a[:, :K].double(), self.w[:, :K].double()
            self.ref = ah @ wh.T + self.a[:, K:].double() @ wh.T + ah @ self.w[:, K:].double().T
        else:
            self.a = pack_a_f8(A, S_A)
            self.w = torch.zeros(N, 4 * K, device="cuda", dtype=torch.uint8)
            self.w_inv = torch.zeros(N, device="cuda")
            _lib.check(lib.pg_pack_weight(W.data_ptr(), N, K, 2, self.w.data_ptr(), self.w_inv.data_ptr(), None))
            torch.cuda.synchronize()
            t = 1.0 / self.w_inv.double()
            whi = self.w[:, :2 * K].contiguous().view(torch.float16).double()
            whi8 = dq8(self.w[:, 2 * K:3 * K].contiguous()) / t[:, None]
            wlo8 = dq8(self.w[:, 3 * K:].contiguous()) / (2048.0 * t[:, None])
            ahi, alo8, ahi8 = unpack_f8(self.a, K, S_A)
            self.ref = ahi @ whi.T + alo8 @ whi8.T + ahi8 @ wlo8.T
        self.ld = K if nseg == 1 else 2 * K


def run_gemm(op, epi, out_fmt=0, bias=True, resid=None, rot=None, **form):
    """One pg_gemm_form launch -> the output buffer (epi 2: the updated copy of `resid`; epi 7: None). rot = (cos, sin, T, dim)."""
    lib = _lib.load()
    a = _lib.PgGemmArgs()
    a.a, a.lda, a.w, a.ldw = op.a.data_ptr(), op.ld, op.w.data_ptr(), op.ld
    a.bias = op.bias.data_ptr() if bias else None
    a.M, a.N, a.K, a.nseg, a.epi = op.M, op.N, op.K, op.nseg, epi
    if op.nseg == 2:
        a.a_scale, a.w_inv = S_A, op.w_inv.data_ptr()
    out = None
    if epi == 2:
        out = resid.clone()
        a.resid, a.ldr = out.data_ptr(), op.N
    elif epi != 7:
        n = op.N // 2 if epi == 5 else op.N
        if out_fmt == 2:
            out = torch.full((op.M, 4 * n), 0xFF, device="cuda", dtype=torch.uint8)
        else:
            out = torch.full((op.M, n * (2 if out_fmt else 1)), float("nan"), device="cuda", dtype=torch.float16)
        a.out_h, a.ldo, a.out_lo_off = out.data_ptr(), (2 * n if out_fmt else n), (n if out_fmt else 0)
        a.out_fmt, a.out_scale = out_fmt, (S_OUT if out_fmt == 2 else 0.0)
    if rot is not None:
        a.rot_cos, a.rot_sin, a.rot_T, a.rot_dim = rot[0].data_ptr(), rot[1].data_ptr(), rot[2], rot[3]
    f = _lib.PgGemmForm()
    for k, v in form.items():
        setattr(f, k, v)
    _lib.check(lib.pg_gemm_form(C.byref(a), C.byref(f), None))
    torch.cuda.synchronize()
    return out


def gemm_values(out, n, out_fmt, epi):
    if epi == 2:
        return out.double()
    if out_fmt == 2:
        hi, lo8, _ = unpack_f8(out, n, S_OUT)
        return hi + lo8
    o = out.view(torch.float16) if out.dtype == torch.uint8 else out
    return o[:, :n].double() + (o[:, n:2 * n].double() if out_fmt == 1 else 0)


def act_ref(x, epi):
    if epi == 1:
        return x * 0.5 * (1 + torch.erf(x / 2 ** 0.5))
    if epi == 4:
        return torch.relu(x) ** 2
    if epi == 6:
        return x * 0.5 * (1 + torch.tanh(0.79788456 * x * (1 + 0.044715 * x * x)))
    if epi == 5:  # w rows interleaved in blocks of 8: gate columns 16i + c, up columns 16i + 8 + c -> output column 8i + c
        v = x.view(x.shape[0], -1, 2, 8)
        return (torch.nn.functional.silu(v[:, :, 0]) * v[:, :, 1]).reshape(x.shape[0], -1)
    return x


def rotate(x, cos, sin, pos, dim, half):
    """rotate-half rotary over slots of 2 * half columns in the first 2 * dim columns; row i at table row pos[i]."""
    c, s = cos[pos].double(), sin[pos].double()
    r = x.clone()
    for h0 in range(0, 2 * dim, 2 * half):
        x1, x2 = x[:, h0:h0 + half], x[:, h0 + half:h0 + 2 * half]
        r[:, h0:h0 + half], r[:, h0 + half:h0 + 2 * half] = x1 * c - x2 * s, x2 * c + x1 * s
    return r


def acc_bound(lmax, xmax):
    """Accumulation error of the pre-activation values against fp64 of the planes. The tensor core truncates while it accumulates one
    hi*hi piece of lmax elements along K (the pieces are then added in round-to-nearest fp32), so the error grows with the longest
    piece: measured on an H100 80GB HBM3 (700 W) at 1.2e-9 .. 3.4e-9 * lmax * max(4, max|x|) for lmax = 64 .. 1280 (epilogues 0-7,
    nseg 1-3, both CTA forms); bound 4e-9 * lmax, plus 2^-23 for the final fp32 rounding of small K."""
    return (4e-9 * lmax + 2.0 ** -23) * max(4.0, xmax)


def gemm_bound(K, xmax, omax, out_fmt, epi=0):
    """acc_bound (K <= the default 1280-element chunk: one piece) times the activation's measured slope, plus the rounding of the
    output planes: fp16 hi alone 2^-11 relative, the e4m3 low plane 2^-16 (test_gemm_f16f8_matches_fp64)."""
    slope = {1: 1.13, 4: max(1.0, xmax), 5: 2.0, 6: 1.13}.get(epi, 1.0)
    rnd = {0: 2.0 ** -11 * max(1.0, omax), 1: 0.0, 2: 2.0 ** -16 * max(1.0, omax)}[0 if epi == 2 else out_fmt]
    return slope * acc_bound(K, xmax) + rnd


def with_knobs(fn, **knobs):
    lib = _lib.load()
    try:
        for k, v in knobs.items():
            lib.pg_set_tuning(k.encode(), v)
        return fn()
    finally:
        lib.pg_set_tuning(b"gemm_cta2", CTA2_DEFAULT)
        lib.pg_set_tuning(b"gemm_prefetch", PREFETCH_DEFAULT)
        lib.pg_set_tuning(b"gemm_kchunk", KCHUNK_DEFAULT)


@pytest.mark.parametrize("nseg", [1, 2, 3])
@pytest.mark.parametrize("cta2", [0, 1])
def test_rotary_positions_per_row(cta2, nseg):
    """Epilogue 3 with rot_pos (PoET: positions that restart in every sequence), M = 300 (not a multiple of 128): segment-restart
    positions and a non-monotone permutation against fp64; rot_pos = arange(M) % rot_T equals rot_pos = NULL bit for bit."""
    M, N, K, rT, dim = 300, 384, 128, 160, 128
    op = GemmOp(M, N, K, nseg, seed=nseg)
    g = torch.Generator(device="cuda").manual_seed(3)
    cos, sin = torch.rand(rT, 32, device="cuda", generator=g), torch.rand(rT, 32, device="cuda", generator=g)
    rot = (cos, sin, rT, dim)
    fmt = 0 if nseg == 1 else (2 if nseg == 2 else 1)
    restart = torch.cat([torch.arange(n) for n in (37, 100, 1, 64, 98)]).to(torch.int32).cuda()
    perm = torch.randperm(M, generator=torch.Generator().manual_seed(1)).to(torch.int32).cuda() % rT
    worst, bound = 0.0, 0.0
    for pos in (restart, perm):
        out = with_knobs(lambda: run_gemm(op, 3, fmt, rot=rot, rot_pos=pos.data_ptr()), gemm_cta2=cta2)
        x = op.ref + op.bias.double()
        ref = rotate(x, cos, sin, pos.long(), dim, 32)
        worst = max(worst, (gemm_values(out, N, fmt, 3) - ref).abs().max().item())
        bound = max(bound, gemm_bound(K, x.abs().max().item(), ref.abs().max().item(), fmt))
    mod = (torch.arange(M, device="cuda") % rT).to(torch.int32)
    a = with_knobs(lambda: run_gemm(op, 3, fmt, rot=rot, rot_pos=mod.data_ptr()), gemm_cta2=cta2)
    b = with_knobs(lambda: run_gemm(op, 3, fmt, rot=rot), gemm_cta2=cta2)
    assert same_bits(a, b)
    report(f"epi 3 rot_pos nseg {nseg} cta2 {cta2}", worst, bound)


@pytest.mark.parametrize("dim", [128, 256])
@pytest.mark.parametrize("nseg", [1, 2, 3])
@pytest.mark.parametrize("cta2", [0, 1])
def test_rotary_128_wide_slots(cta2, nseg, dim):
    """Epilogue 3 with rot_half = 64 (ProGen2's 128-wide head slots): column c and c + 64 of each slot pair up, tables [T, 64] with
    ProGen2's cos = 1, sin = 0 past rotary_dim / 2 (here rotary_dim = 64: the first 32 columns rotate)."""
    M, N, K, rT = 300, 3 * dim, 128, 37
    op = GemmOp(M, N, K, nseg, seed=dim + nseg)
    g = torch.Generator(device="cuda").manual_seed(4)
    ang = torch.rand(rT, 64, device="cuda", generator=g) * 6.0
    ang[:, 32:] = 0.0
    cos, sin = torch.cos(ang), torch.sin(ang)
    fmt = 0 if nseg == 1 else (2 if nseg == 2 else 1)
    out = with_knobs(lambda: run_gemm(op, 3, fmt, rot=(cos, sin, rT, dim), rot_half=64), gemm_cta2=cta2)
    x = op.ref + op.bias.double()
    ref = rotate(x, cos, sin, torch.arange(M, device="cuda") % rT, dim, 64)
    report(f"epi 3 rot_half 64 dim {dim} nseg {nseg} cta2 {cta2}", (gemm_values(out, N, fmt, 3) - ref).abs().max().item(),
           gemm_bound(K, x.abs().max().item(), ref.abs().max().item(), fmt))


W_UNIFORM_CASES = [(e, f) for e in (0, 1, 3, 4, 5, 6) for f in (0, 1, 2)] + [(2, 0)]


@pytest.mark.parametrize("epi,out_fmt", W_UNIFORM_CASES)
@pytest.mark.parametrize("cta2", [0, 1])
def test_f16f8_one_scale_per_matrix(cta2, epi, out_fmt):
    """nseg 2 with w_uniform = 1 (every model's f16f8 linear layers: one e4m3 scale per weight matrix, as pg_pack_weight fmt 2 writes)
    against fp64 of the planes, with test_gemm_f16f8_matches_fp64's bound, and bit-identical to the per-column branch."""
    M, N, K = 300, 384, 256
    op = GemmOp(M, N, K, 2, seed=epi * 3 + out_fmt)
    g = torch.Generator(device="cuda").manual_seed(5)
    resid = torch.randn(M, N, device="cuda", generator=g) if epi == 2 else None
    rot = None
    x = op.ref + op.bias.double()
    if epi == 3:
        cos, sin = torch.rand(37, 32, device="cuda", generator=g), torch.rand(37, 32, device="cuda", generator=g)
        rot = (cos, sin, 37, 128)
    out = with_knobs(lambda: run_gemm(op, epi, out_fmt, resid=resid, rot=rot, w_uniform=1), gemm_cta2=cta2)
    per_col = with_knobs(lambda: run_gemm(op, epi, out_fmt, resid=resid, rot=rot), gemm_cta2=cta2)
    assert same_bits(out, per_col)
    ref = act_ref(x, epi)
    if epi == 2:
        ref = ref + resid.double()
    if epi == 3:
        ref = rotate(x, cos, sin, torch.arange(M, device="cuda") % 37, 128, 32)
    n = N // 2 if epi == 5 else N
    report(f"f16f8 w_uniform epi {epi} out_fmt {out_fmt} cta2 {cta2}", (gemm_values(out, n, out_fmt, epi) - ref).abs().max().item(),
           gemm_bound(K, x.abs().max().item(), ref.abs().max().item(), out_fmt, epi))


@pytest.mark.parametrize("nseg", [1, 2, 3])
@pytest.mark.parametrize("cta2", [0, 1])
def test_per_launch_kchunk(cta2, nseg):
    """A launch's own K chunk (PoET: 64) equals, bit for bit, the same chunk set process-wide; at K = 4096 the 64 k-blocks are cut into
    22 pieces at most (the segment table's cap), 3 k-blocks for the longest, and the error against fp64 follows the longest piece."""
    M, N, K = 300, 320, 4096
    op = GemmOp(M, N, K, nseg, seed=40 + nseg)
    resid = torch.randn(M, N, device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
    form = with_knobs(lambda: run_gemm(op, 2, resid=resid, kchunk=64), gemm_cta2=cta2)
    knob = with_knobs(lambda: run_gemm(op, 2, resid=resid), gemm_cta2=cta2, gemm_kchunk=64)
    assert same_bits(form, knob)
    dflt = with_knobs(lambda: run_gemm(op, 2, resid=resid), gemm_cta2=cta2)
    ref = op.ref + op.bias.double() + resid.double()
    err, err_dflt = (form.double() - ref).abs().max().item(), (dflt.double() - ref).abs().max().item()
    bound = acc_bound(3 * 64, (op.ref + op.bias.double()).abs().max().item())  # 64 k-blocks in 22 pieces: the longest holds 3
    print(f"\n[kernel forms] K=4096 kchunk 64 nseg {nseg}: {err:.3e}; default kchunk 1280: {err_dflt:.3e}")
    report(f"kchunk 64 K=4096 nseg {nseg} cta2 {cta2}", err, bound)


def lm_inputs(B, T, N):
    """ids [B*T] with next-token targets in the first tile, the last (81-column) tile, column N - 1 and odd columns of every lane
    position, and lens that leave rows with t + 1 >= lens."""
    rng = np.random.RandomState(7)
    ids = rng.randint(0, N, size=B * T)
    special = [0, 1, 7, 8, 127, 128, 129, N - 81, N - 2, N - 1, 12345, 12347, 4099, 50001]
    ids[1:1 + len(special)] = special
    lens = np.array([T, 17, 1][:B] + [T] * max(0, B - 3))
    return torch.tensor(ids, dtype=torch.int32, device="cuda"), torch.tensor(lens, dtype=torch.int32, device="cuda"), lens


@pytest.mark.parametrize("K", [64, 1280])
@pytest.mark.parametrize("nseg", [1, 3])
@pytest.mark.parametrize("cta2", [0, 1])
def test_lm_head_partials(cta2, nseg, K):
    """Epilogue 7 (ProtGPT2's 50 257-way head, odd N, last tile 81 columns wide): per (row, tile) max and sum exp, the target logit and
    the logits against fp64; rows with t + 1 >= lens leave every buffer untouched; the partials combined in fp64 give log_softmax."""
    N, B, T = 50257, 3, 50
    M, tiles = B * T, (N + 127) // 128
    op = GemmOp(M, N, K, nseg, seed=K + nseg, a_gain=4.0)
    ids, lens, lens_h = lm_inputs(B, T, N)
    SENT = -1234.5
    part = torch.full((M, tiles, 2), SENT, device="cuda")
    tgt = torch.full((M,), SENT, device="cuda")
    logits = torch.full((M, N), SENT, device="cuda")
    with_knobs(lambda: run_gemm(op, 7, bias=False, lm_part=part.data_ptr(), lm_tgt=tgt.data_ptr(), lm_logits=logits.data_ptr(),
                                lm_ids=ids.data_ptr(), lm_lens=lens.data_ptr(), lm_T=T), gemm_cta2=cta2)
    live = torch.tensor([(r % T) + 1 < lens_h[r // T] for r in range(M)], device="cuda")
    assert (part[~live] == SENT).all() and (tgt[~live] == SENT).all() and (logits[~live] == SENT).all()
    L = op.ref[live]
    pad = torch.full((L.shape[0], tiles * 128 - N), float("-inf"), device="cuda", dtype=torch.float64)
    Lt = torch.cat([L, pad], 1).view(-1, tiles, 128)
    m_ref = Lt.max(-1).values
    se_ref = torch.exp(Lt - m_ref[..., None]).sum(-1)
    m, se = part[live][..., 0].double(), part[live][..., 1].double()
    rows = torch.nonzero(live).flatten()
    lab = ids.long()[rows + 1]
    xmax = L.abs().max().item()
    bound = acc_bound(K, xmax)
    e_logit = (logits[live].double() - L).abs().max().item()
    e_tgt = (tgt[live].double() - L.gather(1, lab[:, None]).flatten()).abs().max().item()
    e_m = (m - m_ref).abs().max().item()
    e_se = ((se - se_ref) / se_ref).abs().max().item()
    lse = torch.logsumexp(m + torch.log(se), -1)
    logp = tgt[live].double() - lse
    e_lp = (logp - torch.log_softmax(L, -1).gather(1, lab[:, None]).flatten()).abs().max().item()
    print(f"\n[kernel forms] epi 7 N={N} K={K} nseg {nseg} cta2 {cta2}: logits {e_logit:.3e} target {e_tgt:.3e} tile max {e_m:.3e} "
          f"tile sum exp (relative) {e_se:.3e} log p {e_lp:.3e}")
    report("epi 7 logits, target, tile max", max(e_logit, e_tgt, e_m), bound)
    # the relative error of a tile's sum of exp is a weighted mean of logit-error differences: half the logit bound (measured 1.4e-6
    # .. 1.6e-5, 2.3 .. 3.8x under); log p = target - logsumexp of the combined partials stays within the logit bound
    report("epi 7 sum exp (relative)", e_se, bound / 2)
    report("epi 7 log p", e_lp, bound)


KNOB_CASES = [(e, n) for e in range(8) for n in (1, 2, 3)]


@pytest.mark.parametrize("epi,nseg", KNOB_CASES)
def test_gemm_knobs_do_not_change_results(epi, nseg):
    """gemm_cta2 x gemm_prefetch only change which CTA computes a tile and when its operands are fetched: every output element has one
    owner and a fixed chunk order, so every combination must give the same bits."""
    M, N, K, T = 300, 384, 256, 100
    op = GemmOp(M, N, K, nseg, seed=epi * 4 + nseg)
    g = torch.Generator(device="cuda").manual_seed(8)
    fmt = 0 if nseg == 1 else (2 if nseg == 2 else 1)
    kw = {}
    if epi == 2:
        kw["resid"] = torch.randn(M, N, device="cuda", generator=g)
    if epi == 3:
        kw["rot"] = (torch.rand(37, 32, device="cuda", generator=g), torch.rand(37, 32, device="cuda", generator=g), 37, 128)
    if op.nseg == 2:
        kw["w_uniform"] = 1
    ids, lens, _ = lm_inputs(3, T, N)

    def once():
        if epi != 7:
            return run_gemm(op, epi, fmt, **kw)
        part = torch.zeros(M, 3, 2, device="cuda")
        tgt = torch.zeros(M, device="cuda")
        logits = torch.zeros(M, N, device="cuda")
        run_gemm(op, 7, bias=False, lm_part=part.data_ptr(), lm_tgt=tgt.data_ptr(), lm_logits=logits.data_ptr(),
                 lm_ids=ids.data_ptr(), lm_lens=lens.data_ptr(), lm_T=T, **kw)
        return torch.cat([part.flatten(), tgt, logits.flatten()])

    outs = [with_knobs(once, gemm_cta2=c, gemm_prefetch=p) for c in (0, 1) for p in (0, 4)]
    assert all(same_bits(o, outs[0]) for o in outs[1:])
