"""PoET host logic without a GPU: the sampler, the a3m read, the encoding, the CLI surface and the loader against the committed goldens
(tests/golden/poet_goldens.jsonl, written by oracle/gen_golden_poet.py from the unmodified reference)."""
import json
import os
import re

import numpy as np
import pytest
import torch

from proteingym_b200 import checkpoint, synth
from proteingym_b200 import poet_engine as E
from proteingym_b200.score_poet import create_parser

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "poet_goldens.jsonl")
CASES = [json.loads(ln) for ln in open(GOLDEN)]


def _bruteforce_neighbors(msa):
    masked = np.where(msa == E.GAP, 255, msa)
    sim = (msa[:, None, :] == masked[None, :, :]).sum(axis=2) / (msa != E.GAP).sum(axis=1, keepdims=True)
    return ((1 - sim) <= E.THETA).sum(axis=1)


@pytest.mark.parametrize("case", [c for c in CASES if "idxs" in c["sampler"]], ids=lambda c: c["name"])
def test_sampler_matches_reference(case):
    seqs = [r.encode() for r in case["a3m"]]
    msa = E.weight_matrix(seqs)
    nb = _bruteforce_neighbors(msa)
    seed = int(case["flags"][case["flags"].index("--seed") + 1])
    ctx = [int(x) for x in case["flags"][1:case["flags"].index("--seed")]]
    for sim in E.SIMILARITIES:
        idx = E.sample_idxs(msa, nb, sim, seed)
        assert idx.tolist() == case["sampler"]["idxs"][str(sim)]
        for mt in ctx:
            lens = [len(s) for s in E.sample_context(seqs, idx, mt, seed)]
            assert lens == case["sampler"]["ctx_lens"][f"{mt}:{sim}"]


def test_min_matches_brute_force():
    n = np.arange(1, 3000)
    got = E.min_matches(n)
    for k, m in zip(n.tolist(), got.tolist()):
        ok = [mm for mm in range(k + 1) if 1 - mm / k <= E.THETA]
        assert m == ok[0]


def test_all_gap_row_fails_like_reference():
    case = next(c for c in CASES if c["name"] == "fail_all_gap_row")
    assert case["error"].startswith("AssertionError") and case["sampler"]["error"].startswith("AssertionError")
    with pytest.raises(AssertionError):
        E.neighbor_counts(E.weight_matrix([r.encode() for r in case["a3m"]]))


def test_encoding_and_a3m_parse():
    assert E.encode(b"ARNDCQEGHILKMFPSTWYV").tolist() == list(range(20))
    assert E.encode(b"-*$XOUBZJa.").tolist() == [20, 21, 22, 23, 11, 4, 23, 23, 23, 23, 23]
    data = b"# comment\n>wt\nACD\nEF\n>h1 desc\nA-dD\n EF \n>h2\n"
    seqs = E.parse_a3m(data)
    assert seqs == [b"ACDEF", b"A-dDEF", b""]
    assert E.weight_matrix(seqs[:2]).tolist() == [E.encode(b"ACDEF").tolist(), E.encode(b"A-DEF").tolist()]
    assert E.context_sequence(b"A-dDEF") == b"ADDEF"  # insertions kept (upper-cased), gaps deleted


def test_zstd_plain_and_magic(tmp_path):
    p = tmp_path / "x.a3m.zst"
    p.write_bytes(b">a\nAC\n")
    assert E.read_maybe_zstd(str(p)) == b">a\nAC\n"
    p.write_bytes(E.ZSTD_MAGIC + b"\x00" * 8)
    try:
        import pyzstd  # noqa: F401
        have = True
    except ImportError:
        try:
            import zstandard  # noqa: F401
            have = True
        except ImportError:
            have = False
    if not have:
        with pytest.raises(RuntimeError, match="pyzstd or zstandard"):
            E.read_maybe_zstd(str(p))


def test_reverse_swaps_start_and_stop():
    row = E.append_startstop(E.encode(b"ACD"))
    rev = E.reverse([row])[0]
    assert rev[0] == E.STOP and rev[-1] == E.START and rev[1:-1].tolist() == E.encode(b"DCA").tolist()


def test_cli_flags_match_reference():
    ref = json.load(open(os.path.join(ROOT, "tests", "golden", "poet_cli_flags.json")))["actions"]
    ours = {a.dest: a for a in create_parser()._actions}
    for r in ref:
        a = ours[r["dest"]]
        assert a.option_strings == r["option_strings"] and a.default == r["default"] and a.nargs == r["nargs"]
        assert getattr(a.type, "__name__", None) == r["type"]
    assert set(ours) - {r["dest"] for r in ref} == {"help", "precision", "device"}


def test_loader_refusals(tmp_path):
    p = str(tmp_path / "c.ckpt")
    synth.write_poet_checkpoint(p, synth.PoetArch(1, 128, 2))
    conf, st = checkpoint.load_poet_checkpoint(p)
    assert (conf.layers, conf.hidden_dim, conf.heads, conf.ff_dim, conf.norm) == (1, 128, 2, 512, False)
    assert "decoder.layers.0.self_attn.q_proj.weight" in st and "norm.weight" not in st
    ck = torch.load(p, weights_only=True)
    for change, msg in [(dict(nhead=4), "head_dim"), (dict(use_multi_rotary=False), "use_multi_rotary"), (dict(n_vocab=25), "n_vocab")]:
        c2 = dict(ck, hyper_parameters={"model_spec": {"init_args": dict(ck["hyper_parameters"]["model_spec"]["init_args"], **change)}})
        q = str(tmp_path / "bad.ckpt")
        torch.save(c2, q)
        with pytest.raises(NotImplementedError, match=msg):
            checkpoint.load_poet_checkpoint(q)


def test_rotary_tables_pair_columns():
    inv = synth.make_poet_state(synth.PoetArch(1, 128, 2))["rotary_emb.inv_freq"]
    cos, sin = E.rotary_tables(inv, 5)
    assert cos.shape == (5, 32)
    assert torch.allclose(cos[3, 1], torch.cos(torch.tensor(3.0) * inv[2]))


def test_header_has_poet_arch():
    hdr = open(os.path.join(ROOT, "include", "pgscore.h")).read()
    assert re.search(r"PG_ARCH_POET\s*=\s*8", hdr)
    assert "int pg_poet_context(" in hdr and "int pg_poet_loglik(" in hdr


def _oracle_scores(case, dtype=torch.float64, device="cpu"):
    """The reference's ensemble on the fp64 oracle: host sampler, oracle context record and per-token log p, float32 averaging."""
    import sys
    sys.path.insert(0, ROOT)
    from oracle.poet_oracle import PoetOracle
    arch = synth.PoetArch(**case["arch"])
    orc = PoetOracle(synth.make_poet_state(arch, seed=case["seed"]), arch.layers, arch.heads, dtype, device)
    seqs = [r.encode() for r in case["a3m"]]
    msa = E.weight_matrix(seqs)
    nb = _bruteforce_neighbors(msa)
    f = case["flags"]
    seed = int(f[f.index("--seed") + 1])
    ctx_lens = [int(x) for x in f[1:f.index("--seed")]]
    wt = case["ref"]["target_seq"][case["ref"]["MSA_start"] - 1:case["ref"]["MSA_end"]]
    variants = [E.append_startstop(E.encode(v.encode())) for v in case["variants"]]
    if "--relative_to_wt" in f:
        variants.append(E.append_startstop(E.encode(wt.encode())))
    logps = []
    for mt in ctx_lens:
        for sim in E.SIMILARITIES:
            ctx = E.sample_context(seqs, E.sample_idxs(msa, nb, sim, seed), mt, seed)
            both = []
            for rows, var in ((ctx, variants), (E.reverse(ctx), E.reverse(variants))):
                rec = orc.context(torch.from_numpy(np.concatenate(rows)).long(), [len(r) for r in rows]) if rows else []
                both.append(np.array([float(orc.token_logp(torch.from_numpy(v).long(), rec).sum()) for v in var], dtype=np.float32))
            logps.append((both[0] + both[1]) / 2)
    s = np.vstack(logps).mean(axis=0)
    return s[:-1] - s[-1] if "--relative_to_wt" in f else s


@pytest.mark.parametrize("case", [c for c in CASES if "scores" in c and c["name"] not in ("long_context", "poet_true_shape")],
                         ids=lambda c: c["name"])
def test_oracle_matches_reference_goldens(case):
    got = _oracle_scores(case)
    assert np.abs(got - np.array(case["scores"])).max() <= 1e-3
