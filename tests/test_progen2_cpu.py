"""CPU: ProGen2 host logic against the goldens of the unmodified reference (oracle/gen_golden_progen2.py): the fp32 oracle reproduces the
reference's scores, the tokenizer matches the reference tokenizer's encodings, the chunk plan and its NaN / failure edges, the library's
head-slot placement of the fused q / v / k projection, the checkpoint loader's key mapping, dtypes and refusals, and the drop-in CLI's
flags."""
import json
import os

import numpy as np
import pandas as pd
import pytest
import torch

from oracle import progen2_oracle as O
from proteingym_b200 import checkpoint, synth
from proteingym_b200.progen2_engine import Progen2Tokenizer, target_row
from proteingym_b200.rita_engine import chunks, plan
from proteingym_b200.tranception_engine import apply_substitutions

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(GOLDEN, "progen2_goldens.jsonl")) as _fh:
    RECORDS = [json.loads(line) for line in _fh]
CASES = {r["name"]: r for r in RECORDS if r["kind"] == "case"}


def _names(ok, true_size=False):
    return [n for n, c in CASES.items() if (c["error"] is None) == ok and c["true_size"] == true_size]


def _seqs(meta):
    dms = pd.DataFrame(meta["dms"])
    if "mutated_sequence" in dms.columns:
        return list(dms["mutated_sequence"])
    return ["1" + apply_substitutions(meta["sequence"], m) + "2" for m in dms["mutant"]]


@pytest.mark.parametrize("name", _names(True))
def test_oracle_reproduces_reference_golden(name):
    meta = CASES[name]
    arch = synth.Progen2Arch(**meta["arch"])
    seqs = _seqs(meta)
    want = np.array(meta["reference_scores"], dtype=np.float64)
    st = synth.make_progen2_state(arch, meta["seed"])
    got = O.calc_fitness(st, seqs, Progen2Tokenizer().encode, arch.heads, arch.rotary_dim, arch.n_positions)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    if np.isfinite(want).any():
        assert np.nanmax(np.abs(got - want)) <= 1e-6
    if name == "wrap_1024":  # the last chunk is one residue and the '2' terminal: no target remains
        assert np.isnan(want).all()


def test_tokenizer_matches_reference_encodings():
    tok = Progen2Tokenizer()
    for c in (r for r in RECORDS if r["kind"] == "encoding"):
        assert tok.encode(c["text"]) == c["ids"], c["text"]
    assert tok.encode("1MKVA2") == [3, 16, 14, 25, 5, 4] and tok.encode("ACJ D") == [5, 7, 8]
    with pytest.raises(NotImplementedError):
        tok.encode("AC<|bos|>D")


def test_target_rows_and_edges():
    assert target_row([3, 5, 6, 4]) == ([3, 5, 6], 2)      # the '2' target is dropped
    assert target_row([4, 6, 5, 3]) == ([4, 6, 5], 2)      # reversed: the '1' target is dropped
    assert target_row([5, 6]) == ([5, 6], 1)
    assert target_row([5, 4]) == ([5], 0)                  # no target left: the reference's mean over nothing, NaN
    for bad in ([], [5], [5, 3, 6]):
        with pytest.raises(ValueError):
            target_row(bad)


@pytest.mark.parametrize("name", _names(False))
def test_failing_goldens_fail_in_the_plan(name):
    """Every case where the reference raised fails before the GPU in the host code too (or in the loader / mutant parsing)."""
    meta = CASES[name]
    if name in ("tiny_rejected", "rotary_none"):
        return  # mutant parsing (apply_substitutions) and the loader: test_cli_parsing_failures / test_loader_refusals
    arch = synth.Progen2Arch(**meta["arch"])
    seqs = _seqs(meta)
    tok = Progen2Tokenizer()
    with pytest.raises(ValueError):
        for s in seqs:
            for c in chunks(s, arch.n_positions):
                target_row(tok.encode(c))
                target_row(tok.encode(c[::-1]))


def test_cli_parsing_failures():
    meta = CASES["tiny_rejected"]
    with pytest.raises(AssertionError) as e:
        for m in meta["dms"]["mutant"]:
            apply_substitutions(meta["sequence"], m)
    assert str(e.value) == meta["error"]["message"]


def test_plan_chunks_and_wild_type_rows():
    assert chunks("A" * 1023, 1024) == ["A" * 1023]
    assert [len(c) for c in chunks("A" * 2050, 1024)] == [1024, 1024, 2]
    assert [len(c) for c in chunks("A" * 2048, 1024)] == [1024, 1024, 0]
    wt = "1" + synth.random_protein(300, 1) + "2"
    mut = wt[:200] + ("A" if wt[200] != "A" else "C") + wt[201:]
    rows, index, wt_of = plan([mut, wt], wt, 1024)
    assert rows[index[1][0]] == wt and rows[index[1][1]] == wt[::-1]
    assert wt_of[index[0][0]] == index[1][0] and wt_of[index[0][1]] == index[1][1]


def test_slot_placement_restated():
    """api.cu slot_src's ProGen2 maps, restated: q / k rows of slot h take the (2i, 2i+1) pairs of head h's shard rows at (Si, S/2 + i);
    with 1/sqrt(hd) on q and rotate-half rotary on the slot pairs, q.k per head equals the reference's rotate_every_two attention."""
    d, heads, rot = 768, 8, 64
    hd, S = d // heads, 128
    g = torch.Generator().manual_seed(1)
    w = torch.randn(3 * d, d, generator=g, dtype=torch.float64)
    x = torch.randn(5, d, generator=g, dtype=torch.float64)
    per = heads // 8

    def src(i, part):
        h, c = divmod(i, S)
        base = (h // per) * (3 * d // 8) + (h % per) * hd
        if part == "v":
            return base + d // 8 + c if c < hd else -1
        off = 0 if part == "q" else 2 * d // 8
        if c < hd // 2:
            return base + off + 2 * c
        if S // 2 <= c < S // 2 + hd // 2:
            return base + off + 2 * (c - S // 2) + 1
        return -1
    wz = torch.cat([w, torch.zeros(1, d, dtype=w.dtype)])
    proj = {p: x @ wz[[src(i, p) for i in range(heads * S)]].T for p in "qkv"}
    sin, cos = (t.double() for t in O.rotary_tables(rot, 5))
    c_t = torch.ones(5, S // 2, dtype=torch.float64)
    s_t = torch.zeros(5, S // 2, dtype=torch.float64)
    c_t[:, :rot // 2], s_t[:, :rot // 2] = cos, sin

    def rope(t):
        t = t.view(5, heads, 2, S // 2)
        a, b = t[:, :, 0], t[:, :, 1]
        return torch.stack((a * c_t[:, None] - b * s_t[:, None], b * c_t[:, None] + a * s_t[:, None]), 2).view(5, heads, S)
    q, k = rope(proj["q"]) / hd ** 0.5, rope(proj["k"])
    ours = torch.einsum("thc,shc->hts", q, k)
    qkv = (x @ w.T).view(5, 8, -1)
    rq, rv, rk = (t.reshape(5, heads, hd) for t in torch.split(qkv, d // 8, -1))
    rq = torch.cat([O._rotate(rq[..., :rot], sin, cos), rq[..., rot:]], -1)
    rk = torch.cat([O._rotate(rk[..., :rot], sin, cos), rk[..., rot:]], -1)
    ref = torch.einsum("thc,shc->hts", rq, rk) / hd ** 0.5
    assert torch.allclose(ours, ref, atol=1e-10)
    assert torch.equal(proj["v"].view(5, heads, S)[..., :hd], rv) and not proj["v"].view(5, heads, S)[..., hd:].any()


def test_loader_key_mapping_dtypes_and_refusals(tmp_path):
    arch = synth.Progen2Arch(2, 512, 8, 32)
    st = synth.write_progen2_checkpoint(str(tmp_path / "m"), arch, seed=2)
    conf, state = checkpoint.load_progen2_checkpoint(str(tmp_path / "m"))
    assert (conf.layers, conf.embed_dim, conf.heads, conf.ffn_dim, conf.vocab, conf.rotary_dim, conf.n_positions) == (2, 512, 8, 2048, 32, 32, 1024)
    assert "h.0.attn.qkv_proj.weight" in state and "lm_head.bias" in state and not any("attn.bias" in k or "masked_bias" in k for k in state)
    assert torch.equal(state["wte.weight"], st["transformer.wte.weight"])
    half = {k: (v.half() if v.dtype.is_floating_point else v) for k, v in st.items()}
    synth.write_progen2_checkpoint(str(tmp_path / "h"), arch, state=half)
    _, sh = checkpoint.load_progen2_checkpoint(str(tmp_path / "h"))
    assert sh["h.1.mlp.fc_in.weight"].dtype == torch.float32
    synth.write_progen2_checkpoint(str(tmp_path / "s"), arch, seed=2, safetensors=True)
    assert checkpoint.load_progen2_checkpoint(str(tmp_path / "s"))[0].layers == 2
    for extra, err, match in (({"layer_norm_epsilon": 1e-6}, NotImplementedError, "eps"), ({"rotary_dim": None}, ValueError, "rotary_dim"),
                              ({"activation_function": "gelu"}, NotImplementedError, "gelu_new")):
        synth.write_progen2_checkpoint(str(tmp_path / "x"), arch, state=st, config_extra=extra)
        with pytest.raises(err, match=match):
            checkpoint.load_progen2_checkpoint(str(tmp_path / "x"))
    xl = synth.Progen2Arch(1, 4096, 16, 64)
    synth.write_progen2_checkpoint(str(tmp_path / "xl"), xl, state={}, config_extra={})
    with pytest.raises(NotImplementedError, match="xlarge"):
        checkpoint.load_progen2_checkpoint(str(tmp_path / "xl"))
    bad = dict(st)
    del bad["transformer.h.1.mlp.fc_out.bias"]
    synth.write_progen2_checkpoint(str(tmp_path / "b"), arch, state=bad)
    with pytest.raises(ValueError, match="fc_out.bias"):
        checkpoint.load_progen2_checkpoint(str(tmp_path / "b"))


def test_cli_flags_match_reference():
    from proteingym_b200 import score_progen2
    want = next(r["flags"] for r in RECORDS if r["kind"] == "cli_flags")
    p = score_progen2.create_parser()
    got = {a.option_strings[0]: a for a in p._actions if a.dest != "help"}
    for flag, spec in want.items():
        a = got[flag]
        assert a.dest == spec["dest"] and a.default == spec["default"] and a.required == spec["required"]
        assert getattr(a.type, "__name__", None) == spec["type"]
    assert set(got) - set(want) == {"--precision", "--device"}
    with pytest.raises(NotImplementedError):
        score_progen2.main(p.parse_args(["--test"]))


def test_refusals_are_in_the_library():
    src = open(os.path.join(GOLDEN, "..", "..", "proteingym_b200", "csrc", "api.cu")).read()
    assert "progen2-xlarge" in src and "ProGen2 needs heads % 8 == 0" in src
    hdr = open(os.path.join(GOLDEN, "..", "..", "include", "pgscore.h")).read()
    assert "PG_ARCH_PROGEN2 = 6" in hdr
