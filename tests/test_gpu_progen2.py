"""GPU: ProGen2 (PG_ARCH_PROGEN2) against the fp64 oracle per predicted token at the small / medium / large widths and head counts (head
dims 64, 96 and 80: 64- and 128-wide head slots), one isolated 128-slot attention layer, exact wild-type prefix reuse, the goldens of the
unmodified reference (oracle/gen_golden_progen2.py) through the drop-in CLI, and refused configurations."""
import ctypes as C
import json
import os

import numpy as np
import pandas as pd
import pytest
import torch

from oracle import progen2_oracle as O
from proteingym_b200 import _lib, checkpoint, synth
from proteingym_b200.progen2_engine import Progen2Scorer

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(GOLDEN, "progen2_goldens.jsonl")) as _fh:
    CASES = {r["name"]: r for r in map(json.loads, _fh) if r["kind"] == "case"}
# fp64 per-token bounds |log p - oracle|: about 4x the worst measured on an H100 80GB HBM3 at 700 W (1.2e-5, 4.6e-5, 1.0e-3; DESIGN.md §2)
BOUND = {"f16x3": 5e-5, "f16f8": 2e-4, "f16": 4e-3}
WIDTHS = {"small": synth.Progen2Arch(2, 1024, 16, 32), "medium": synth.Progen2Arch(2, 1536, 16, 48),
          "large": synth.Progen2Arch(2, 2560, 32, 64)}
TS = (2, 63, 64, 65, 127, 128, 129, 1023)
_CACHE, _ORACLE = {}, {}


def conf_of(a):
    return checkpoint.Progen2Config(a.layers, a.embed_dim, a.heads, a.ffn_dim, a.vocab, a.rotary_dim, a.n_positions)


def weights(st):
    return {k[len("transformer."):] if k.startswith("transformer.") else k: v for k, v in st.items()
            if not (k.endswith("attn.bias") or k.endswith("attn.masked_bias"))}


def scorer(arch, prec, seed=5):
    key = (arch, prec, seed)
    if key not in _CACHE:
        _CACHE.clear()  # one model on the device at a time
        st = synth.make_progen2_state(arch, seed, buffers=False)
        _CACHE[key] = (Progen2Scorer(conf_of(arch), weights(st), precision=prec), st)
    return _CACHE[key]


def oracle_tokens(arch, st, ids):
    key = (arch, tuple(ids))
    if key not in _ORACLE:
        _ORACLE[key] = O.token_logprobs(st, ids, arch.heads, arch.rotary_dim, torch.float64).numpy()
    return _ORACLE[key]


def rows_of(sc, ids):
    """Per-token log p(ids[t+1] | ids[<=t]) of one token row through pg_ar_prefix_begin -> numpy [T-1]."""
    tok, _ = sc.prefix_begin(ids)
    return tok[:len(ids) - 1]


def _ids(rng, T):
    ids = list(rng.randint(5, 30, size=T))
    ids[0] = 3 if T % 2 else ids[0]  # a leading '1' terminal as an input token
    return ids


@pytest.mark.parametrize("width", list(WIDTHS))
@pytest.mark.parametrize("prec", list(BOUND))
def test_tokens_against_fp64(width, prec):
    arch = WIDTHS[width]
    sc, st = scorer(arch, prec)
    rng = np.random.RandomState(7)
    worst, seqs = 0.0, []
    for T in TS:
        ids = _ids(rng, T)
        seqs.append(ids)
        want = oracle_tokens(arch, st, ids)
        got = rows_of(sc, ids)
        worst = max(worst, float(np.abs(got - want).max()))
    sums = sc.token_sums(seqs)  # the ragged batch
    for ids, s in zip(seqs, sums):
        assert abs(s - float(oracle_tokens(arch, st, ids).sum())) <= BOUND[prec] * (len(ids) - 1)
    print(f"ProGen2 {width} (head_dim {arch.head_dim}) {prec}: worst per-token |err| {worst:.3e}")
    assert worst <= BOUND[prec]


@pytest.mark.parametrize("prec", ["f16x3", "f16f8"])
def test_128_slot_attention_layer(prec):
    """One layer, head_dim 96 rotated whole, T = 1023: the attention and rotary of a 128-wide slot carry most of the signal, so a wrong
    pair mapping or a lost second 64-column box moves tokens by orders more than the bound."""
    arch = synth.Progen2Arch(1, 768, 8, 96)
    sc, st = scorer(arch, prec, seed=9)
    ids = _ids(np.random.RandomState(3), 1023)
    err = float(np.abs(rows_of(sc, ids) - oracle_tokens(arch, st, ids)).max())
    print(f"ProGen2 one layer head_dim 96, full rotary, {prec}: worst per-token |err| {err:.3e}")
    assert err <= BOUND[prec]


def _fused_rows(sc, ids_list, start=None):
    """log-probability rows [B, T, 25] of right-padded token rows through pg_ar_loglik_fused (start None) or, after pg_ar_prefix_begin,
    pg_ar_loglik_prefix on the suffixes ids[start:]."""
    sub = [x if start is None else x[start:] for x in ids_list]
    T = max(len(x) for x in sub)
    ids = np.zeros((len(sub), T), dtype=np.int32)
    for r, x in enumerate(sub):
        ids[r, :len(x)] = x
    d_ids = torch.from_numpy(ids).cuda()
    d_lens = torch.tensor([len(x) for x in sub], dtype=torch.int32, device="cuda")
    rows = torch.zeros((len(sub), T, 25), device="cuda")
    out = torch.zeros(len(sub), device="cuda")
    f = _lib.PgArFusion(out_logprobs=rows.data_ptr())
    if start is None:
        rc = sc.lib.pg_ar_loglik_fused(sc.handle, d_ids.data_ptr(), d_lens.data_ptr(), len(sub), T, C.byref(f), out.data_ptr(), None)
    else:
        rc = sc.lib.pg_ar_loglik_prefix(sc.handle, d_ids.data_ptr(), d_lens.data_ptr(), len(sub), T, start, C.byref(f), out.data_ptr(), None)
    _lib.check(rc, sc.handle)
    return rows.cpu().numpy()


@pytest.mark.parametrize("width", ["small", "medium"])
@pytest.mark.parametrize("start", [128, 256])
@pytest.mark.parametrize("reverse", [False, True])
def test_prefix_rows_bit_identical(width, start, reverse):
    sc, st = scorer(WIDTHS[width], "f16f8")
    rng = np.random.RandomState(start + reverse)
    wt = list(rng.randint(5, 30, size=300))
    muts = []
    for k, n in ((start, 300), (start + 1, 300), (start + 30, 290), (299, 300)):
        x = list(wt)
        pos = 299 - k if reverse else k
        x[pos] = 5 + (x[pos] - 4) % 25
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
    csum = np.concatenate([[0.0], np.cumsum(wt_tok.astype(np.float64))])
    got = sc.prefix_suffix_sums(muts, start)
    for m, s, p in zip(muts, got, sc.token_sums(muts)):
        assert abs(csum[start - 1] + float(wt_rows[start - 1, m[start] - 5]) + s - p) <= 2e-5 * abs(p)


def _run_cli(tmp_path, name, prec="f16f8"):
    from proteingym_b200 import score_progen2
    _CACHE.clear()
    meta = CASES[name]
    arch = synth.Progen2Arch(**meta["arch"])
    model = tmp_path / "model"
    synth.write_progen2_checkpoint(str(model), arch, seed=meta["seed"])
    dms = pd.DataFrame(meta["dms"])
    (tmp_path / "dms").mkdir()
    dms.to_csv(tmp_path / "dms" / "ASSAY.csv", index=False)
    pd.DataFrame({"DMS_id": ["ASSAY"], "DMS_filename": ["ASSAY.csv"], "target_seq": [meta["sequence"]]}).to_csv(tmp_path / "ref.csv", index=False)
    (tmp_path / "out").mkdir()
    argv = ["--Progen2_model_name_or_path", str(model), "--DMS_reference_file_path", str(tmp_path / "ref.csv"), "--DMS_data_folder",
            str(tmp_path / "dms"), "--DMS_index", "0", "--output_scores_folder", str(tmp_path / "out"), "--precision", prec]
    if meta["indel_mode"]:
        argv.append("--indel_mode")
    score_progen2.main(score_progen2.create_parser().parse_args(argv))
    return meta, pd.read_csv(tmp_path / "out" / "ASSAY.csv")


def _golden_names(ok):
    return [n for n, c in CASES.items() if (c["error"] is None) == ok]


@pytest.mark.parametrize("name", _golden_names(True))
def test_goldens_within_1e3(tmp_path, name):
    meta, got = _run_cli(tmp_path, name)
    assert list(got.columns) == ["mutant", "Progen2_score", "DMS_score"]
    assert list(got["mutant"]) == meta["dms"]["mutant"]
    g, w = got["Progen2_score"].to_numpy(), np.array(meta["reference_scores"], dtype=np.float64)
    assert np.array_equal(np.isnan(g), np.isnan(w))
    err = float(np.nanmax(np.abs(g - w))) if np.isfinite(w).any() else 0.0
    print(f"ProGen2 golden {name}: max |score - reference| {err:.3e}")
    assert err <= 1e-3


@pytest.mark.parametrize("name", _golden_names(False))
def test_cli_fails_where_reference_fails(tmp_path, name):
    meta = CASES[name]
    with pytest.raises(AssertionError if meta["error"]["type"] == "AssertionError" and name == "tiny_rejected" else ValueError) as e:
        _run_cli(tmp_path, name)
    if name == "tiny_rejected":
        assert str(e.value) == meta["error"]["message"]


def _create(**kw):
    lib = _lib.load()
    d = dict(arch=_lib.PG_ARCH_PROGEN2, layers=2, embed_dim=1024, heads=16, ffn_dim=4096, vocab=32, max_positions=1024, token_dropout=0,
             emb_ln_before=0, precision=_lib.PG_PREC_F16F8, device=0, max_rows=4096)
    d.update(kw)
    h = C.c_void_p()
    rc = lib.pg_create(C.byref(_lib.PgModelDesc(**d)), C.byref(h))
    if rc == 0:
        lib.pg_destroy(h)
    return rc, lib


def test_refused_configurations():
    rc, lib = _create(embed_dim=4096, heads=16, ffn_dim=16384)  # progen2-xlarge
    assert rc == 4 and b"progen2-xlarge" in lib.pg_last_error(None)
    rc, lib = _create(embed_dim=1536, heads=12, ffn_dim=6144)  # head_dim 128, but heads % 8 != 0
    assert rc == 4 and b"heads % 8" in lib.pg_last_error(None)
    rc, lib = _create(precision=_lib.PG_PREC_F16D)
    assert rc == 4 and b"F16D" in lib.pg_last_error(None)
    assert _create(embed_dim=2048, heads=16, ffn_dim=8192)[0] == 0  # head_dim 128 itself is accepted
