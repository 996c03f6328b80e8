"""GPU: RITA (PG_ARCH_RITA) against the fp64 oracle per predicted token, the tanh-GELU GEMM epilogue (epi 6) against fp64, exact wild-type
prefix reuse, the goldens of the unmodified reference (oracle/gen_golden_rita.py), the drop-in CLI end to end, and refused configurations."""
import ctypes as C
import json
import math
import os

import numpy as np
import pandas as pd
import pytest
import torch

from oracle import rita_oracle as O
from proteingym_b200 import _lib, checkpoint, synth
from proteingym_b200.rita_engine import RitaScorer, RitaTokenizer

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# fp64 per-token bounds |log p - oracle|: about 4x the worst measured on an H100 80GB HBM3 at 700 W (1.2e-4, 2.2e-4, 6.1e-3; DESIGN.md §2)
BOUND = {"f16x3": 4.5e-4, "f16f8": 9e-4, "f16": 2.5e-2}
WIDTHS = {"S": synth.RitaArch(2, 768, 12), "M": synth.RitaArch(2, 1024, 16), "L": synth.RitaArch(2, 1536, 24)}
_CACHE = {}


def scorer(arch, prec, seed=5, untied=False, tok="plain"):
    key = (arch, prec, seed, untied, tok)
    if key not in _CACHE:
        st = synth.make_rita_state(arch, seed, untied)
        conf = checkpoint.RitaConfig(arch.layers, arch.embed_dim, arch.heads, arch.ffn_dim, arch.vocab, not untied)
        ws = {k[len("transformer."):] if k.startswith("transformer.") else k: v for k, v in st.items() if "inv_freq" not in k}
        if not untied:
            ws.pop("lm_head.weight")
        inv = st["transformer.layers.0.self_attention.rotary_embedding.inv_freq"]
        _CACHE[key] = (RitaScorer(conf, ws, inv, RitaTokenizer(os.path.join(GOLDEN, f"rita_tokenizer_{tok}")), precision=prec), st)
    return _CACHE[key]


def rows_of(sc, ids):
    """Per-token log p(ids[t+1] | ids[<=t]) of one token row through pg_ar_prefix_begin (it returns the rows) -> numpy [T-1]."""
    tok, _ = sc.prefix_begin(ids)
    return tok[:len(ids) - 1]


@pytest.mark.parametrize("width", list(WIDTHS))
@pytest.mark.parametrize("prec", list(BOUND))
def test_tokens_against_fp64(width, prec):
    arch = WIDTHS[width]
    sc, st = scorer(arch, prec)
    rng = np.random.RandomState(7)
    worst = 0.0
    seqs = []
    for T in (2, 63, 64, 65, 127, 128, 129, 1023):
        ids = list(rng.randint(4, 24, size=T))
        seqs.append(ids)
        want = O.logprob_rows(st, ids, arch.heads, torch.float64)
        want = want[torch.arange(T - 1), torch.as_tensor(ids[1:])].numpy()
        got = rows_of(sc, ids)
        worst = max(worst, float(np.abs(got - want).max()))
        # the plain ragged path gives the same sum as the rows
        assert abs(float(sc.token_sums([ids])[0]) - float(want.sum())) <= BOUND[prec] * (T - 1)
    # a ragged batch: sums against fp64
    sums = sc.token_sums(seqs)
    for ids, s in zip(seqs, sums):
        lp = O.logprob_rows(st, ids, arch.heads, torch.float64)
        ref = float(lp[torch.arange(len(ids) - 1), torch.as_tensor(ids[1:])].sum())
        assert abs(s - ref) <= BOUND[prec] * (len(ids) - 1)
    print(f"RITA {width} {prec}: worst per-token |err| {worst:.3e}")
    assert worst <= BOUND[prec]


@pytest.mark.parametrize("out_fmt", [0, 1, 2])
def test_epi6_gemm_against_fp64(out_fmt):
    lib = _lib.load()
    M, N, K = 200, 384, 256
    g = torch.Generator().manual_seed(3)
    a = torch.randn(M, K, generator=g, dtype=torch.float64)
    w = torch.randn(N, K, generator=g, dtype=torch.float64) / math.sqrt(K) * 3
    b = torch.randn(N, generator=g, dtype=torch.float64)
    want = O.rita_gelu(a @ w.T + b)
    dev = torch.device("cuda")
    nseg = {0: 3, 1: 3, 2: 2}[out_fmt]
    a16 = a.float().to(dev)
    hi = a16.half()
    lo = (a16 - hi.float()).half()
    if nseg == 3:
        a_op = torch.cat([hi, lo], 1).contiguous()
        w_op = torch.empty(N, 2 * K, dtype=torch.half, device=dev)
        _lib.check(lib.pg_pack_weight(w.float().to(dev).data_ptr(), N, K, 1, w_op.data_ptr(), None, None))
        w_inv = None
        a_scale = 0.0
    else:
        a_scale = 4.0
        lo8 = (lo.float() * 2048 * a_scale).to(torch.float8_e4m3fn).view(torch.uint8)
        hi8 = (hi.float() * a_scale).to(torch.float8_e4m3fn).view(torch.uint8)
        a_op = torch.cat([hi.view(torch.uint8).view(M, 2 * K), lo8, hi8], 1).contiguous().view(torch.half)
        w_op = torch.empty(N, 2 * K, dtype=torch.half, device=dev)
        w_inv = torch.empty(N, dtype=torch.float32, device=dev)
        _lib.check(lib.pg_pack_weight(w.float().to(dev).data_ptr(), N, K, 2, w_op.data_ptr(), w_inv.data_ptr(), None))
    out = torch.zeros(M, 2 * N, dtype=torch.half, device=dev)
    bias = b.float().to(dev)
    args = _lib.PgGemmArgs(a=a_op.data_ptr(), lda=2 * K, w=w_op.data_ptr(), ldw=2 * K, bias=bias.data_ptr(), M=M, N=N, K=K, nseg=nseg, epi=6,
                           out_h=out.data_ptr(), ldo=2 * N, out_lo_off=N if out_fmt else 0, a_scale=a_scale,
                           w_inv=w_inv.data_ptr() if w_inv is not None else None, out_fmt=out_fmt, out_scale=2.0)
    _lib.check(lib.pg_gemm(C.byref(args), None))
    torch.cuda.synchronize()
    hi_o = out[:, :N].float()
    if out_fmt == 1:
        got = hi_o + out[:, N:].float()
    elif out_fmt == 2:
        planes = out[:, N:].contiguous().view(torch.uint8)
        got = hi_o + planes[:, :N].view(torch.float8_e4m3fn).float() / (2048 * 2.0)
        assert torch.equal(planes[:, N:2 * N].view(torch.float8_e4m3fn).float(), (hi_o * 2.0).to(torch.float8_e4m3fn).float())
    else:
        got = hi_o
    diff = (got.double().cpu() - want).abs()
    err = diff.max().item()
    print(f"epi 6 out_fmt {out_fmt}: max |err| {err:.3e}")
    if out_fmt == 0:  # one fp16 plane: the rounding of the output itself, half an fp16 ulp
        assert bool((diff <= 2.0 ** -11 * want.abs() + 1e-5).all())
    else:  # measured 6.7e-6 (hi + lo) and 2.1e-4 (hi + e4m3 planes)
        assert err <= {1: 3e-5, 2: 8e-4}[out_fmt]


def _fused_rows(sc, ids_list, start=None):
    """log-probability rows [B, T, vocab] of right-padded token rows through pg_ar_loglik_fused (start None) or, after pg_ar_prefix_begin,
    pg_ar_loglik_prefix on the suffixes ids[start:]."""
    sub = [x if start is None else x[start:] for x in ids_list]
    T = max(len(x) for x in sub)
    ids = np.zeros((len(sub), T), dtype=np.int32)
    for r, x in enumerate(sub):
        ids[r, :len(x)] = x
    d_ids = torch.from_numpy(ids).cuda()
    d_lens = torch.tensor([len(x) for x in sub], dtype=torch.int32, device="cuda")
    rows = torch.zeros((len(sub), T, sc.conf.vocab), device="cuda")
    out = torch.zeros(len(sub), device="cuda")
    f = _lib.PgArFusion(out_logprobs=rows.data_ptr())
    if start is None:
        rc = sc.lib.pg_ar_loglik_fused(sc.handle, d_ids.data_ptr(), d_lens.data_ptr(), len(sub), T, C.byref(f), out.data_ptr(), None)
    else:
        rc = sc.lib.pg_ar_loglik_prefix(sc.handle, d_ids.data_ptr(), d_lens.data_ptr(), len(sub), T, start, C.byref(f), out.data_ptr(), None)
    _lib.check(rc, sc.handle)
    return rows.cpu().numpy()


@pytest.mark.parametrize("start", [128, 256])
@pytest.mark.parametrize("reverse", [False, True])
def test_prefix_rows_bit_identical(start, reverse):
    """Mutants whose first change (in scoring order) is at start, start + 1, start + 60 and the last token, with ragged lengths; R->L
    rows are the reversed strings, whose shared prefix with the reversed wild type ends at the mutant's last change."""
    sc, st = scorer(WIDTHS["S"], "f16f8")
    rng = np.random.RandomState(start + reverse)
    wt = list(rng.randint(4, 24, size=300))
    muts = []
    for k, n in ((start, 300), (start + 1, 300), (start + 30, 290), (299, 300)):
        x = list(wt)
        pos = 299 - k if reverse else k  # protein coordinate of the change
        x[pos] = 4 + (x[pos] - 3) % 20
        if n < 300:
            x = x[:n] if not reverse else x[300 - n:]
        muts.append(x[::-1] if reverse else x)
    w = wt[::-1] if reverse else wt
    assert all(m[:start] == w[:start] for m in muts) and muts[0][start] != w[start]
    plain = _fused_rows(sc, muts)
    wt_tok, wt_rows = sc.prefix_begin(w)
    assert np.array_equal(wt_rows[:299], _fused_rows(sc, [w])[0, :299])
    sfx = _fused_rows(sc, muts, start)
    for r, m in enumerate(muts):
        assert np.array_equal(sfx[r, :len(m) - start - 1], plain[r, start:len(m) - 1])
    # the engine's recombined sums equal the plain sums to fp32 rounding
    csum = np.concatenate([[0.0], np.cumsum(wt_tok.astype(np.float64))])
    got = sc.prefix_suffix_sums(muts, start)
    for m, s, p in zip(muts, got, sc.token_sums(muts)):
        assert abs(csum[start - 1] + float(wt_rows[start - 1, m[start]]) + s - p) <= 2e-5 * abs(p)


def _golden(name):
    with open(os.path.join(GOLDEN, f"rita_{name}_meta.json")) as fh:
        meta = json.load(fh)
    return meta


def _run_cli(tmp_path, name, prec="f16f8"):
    from proteingym_b200 import score_rita
    meta = _golden(name)
    a = meta["arch"]
    arch = synth.RitaArch(a["layers"], a["embed_dim"], a["heads"], a["ff_ratio"], a["vocab"])
    model = tmp_path / "model"
    synth.write_rita_checkpoint(str(model), arch, seed=meta["seed"], untied=meta["untied"])
    dms = pd.read_csv(os.path.join(GOLDEN, f"rita_{name}_dms.csv"))
    (tmp_path / "dms").mkdir()
    dms.to_csv(tmp_path / "dms" / "ASSAY.csv", index=False)
    pd.DataFrame({"DMS_id": ["ASSAY"], "DMS_filename": ["ASSAY.csv"], "target_seq": [meta["sequence"]]}).to_csv(tmp_path / "ref.csv", index=False)
    (tmp_path / "out").mkdir()
    argv = ["--RITA_model_name_or_path", str(model), "--DMS_reference_file_path", str(tmp_path / "ref.csv"), "--DMS_data_folder",
            str(tmp_path / "dms"), "--DMS_index", "0", "--output_scores_folder", str(tmp_path / "out"),
            "--RITA_tokenizer_path", os.path.join(GOLDEN, f"rita_tokenizer_{meta['tokenizer']}"), "--precision", prec]
    if meta["indel_mode"]:
        argv.append("--indel_mode")
    score_rita.main(score_rita.create_parser().parse_args(argv))
    return meta, pd.read_csv(tmp_path / "out" / "ASSAY.csv")


GOLDEN_OK = ["tiny", "tiny_bos", "tiny_untied", "indels", "long_1100", "long_2047", "long_2046_bos", "rita_s", "rita_l"]


@pytest.mark.parametrize("name", GOLDEN_OK)
def test_goldens_within_1e3(tmp_path, name):
    meta, got = _run_cli(tmp_path, name)
    want = pd.read_csv(os.path.join(GOLDEN, f"rita_{name}_reference_output.csv"))
    assert list(got.columns) == ["mutant", "RITA_score", "DMS_score"] == list(want.columns)
    assert list(got["mutant"]) == list(want["mutant"])
    g, w = got["RITA_score"].to_numpy(), want["RITA_score"].to_numpy()
    assert np.array_equal(np.isnan(g), np.isnan(w))
    if name == "long_2047":
        assert np.isnan(w).all()
    err = float(np.nanmax(np.abs(g - w))) if np.isfinite(w).any() else 0.0
    print(f"RITA golden {name}: max |score - reference| {err:.3e}")
    assert err <= 1e-3


@pytest.mark.parametrize("name", ["tiny_rejected", "long_2046"])
def test_cli_fails_where_reference_fails(tmp_path, name):
    meta = _golden(name)
    assert meta["error"] is not None
    with pytest.raises(AssertionError if meta["error"]["type"] == "AssertionError" else ValueError) as e:
        _run_cli(tmp_path, name)
    if meta["error"]["type"] == "AssertionError":
        assert str(e.value) == meta["error"]["message"]


def test_prefix_reuse_changes_nothing_but_work(tmp_path, monkeypatch):
    meta, on = _run_cli(tmp_path, "rita_s")
    monkeypatch.setattr(RitaScorer, "prefix_reuse", False)
    (tmp_path / "off").mkdir()
    _, off = _run_cli(tmp_path / "off", "rita_s")
    assert np.abs(on["RITA_score"].to_numpy() - off["RITA_score"].to_numpy()).max() <= 1e-4


def _create(**kw):
    lib = _lib.load()
    d = dict(arch=_lib.PG_ARCH_RITA, layers=2, embed_dim=128, heads=2, ffn_dim=512, vocab=26, max_positions=1023, token_dropout=0,
             emb_ln_before=0, precision=_lib.PG_PREC_F16F8, device=0, max_rows=4096)
    d.update(kw)
    desc = _lib.PgModelDesc(**d)
    h = C.c_void_p()
    rc = lib.pg_create(C.byref(desc), C.byref(h))
    return rc, h, lib


def test_refused_configurations():
    rc, h, lib = _create(embed_dim=2048, heads=16, ffn_dim=8192)
    assert rc == 4 and b"RITA XL" in lib.pg_last_error(None)
    rc, h, lib = _create(precision=_lib.PG_PREC_F16D)
    assert rc == 4 and b"F16D" in lib.pg_last_error(None)
    sc, _ = scorer(WIDTHS["S"], "f16f8")
    ids = torch.full((1, 8), 5, dtype=torch.int32, device="cuda")
    lens = torch.full((1,), 8, dtype=torch.int32, device="cuda")
    out = torch.zeros(1, device="cuda")
    prior = torch.zeros(8, 26, device="cuda")
    prow = torch.zeros(1, 8, dtype=torch.int32, device="cuda")
    f = _lib.PgArFusion(log_prior=prior.data_ptr(), prior_row=prow.data_ptr(), alpha=0.5)
    assert sc.lib.pg_ar_loglik_fused(sc.handle, ids.data_ptr(), lens.data_ptr(), 1, 8, C.byref(f), out.data_ptr(), None) == 1
    assert b"retrieval" in sc.lib.pg_last_error(sc.handle)
    tok = torch.zeros(8, device="cuda")
    assert sc.lib.pg_ar_prefix_begin(sc.handle, ids.data_ptr(), 8, C.byref(f), tok.data_ptr(), None) == 1
    pos = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert sc.lib.pg_masked_marginals(sc.handle, ids.data_ptr(), 8, pos.data_ptr(), None, None, 1, 8, out.data_ptr(), None) == 3
