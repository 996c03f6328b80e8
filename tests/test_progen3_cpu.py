"""CPU: the ProGen3 fp64 oracle against the goldens of the unmodified reference (oracle/gen_golden_progen3.py), the encoding of both
directions, the FASTA reader, config parsing and refusals (host and pg_create), the megablocks / eager layout equivalence, the drop-in's
flags against the reference's, and that the product path never imports the oracle."""
import ctypes as C
import io
import json
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest
import torch

from oracle import progen3_oracle as O
from proteingym_b200 import _lib, checkpoint, synth
from proteingym_b200.progen3_engine import Progen3Tokenizer, read_fasta

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
with open(os.path.join(GOLDEN, "progen3_goldens.jsonl")) as _fh:
    GOLDENS = {r["name"]: r for r in map(json.loads, _fh)}


def conf_state(arch, seed):
    conf = checkpoint.progen3_config(arch.config())
    return conf, checkpoint.normalise_progen3_state(conf, synth.make_progen3_state(arch, seed))


@pytest.mark.parametrize("name", [n for n, g in GOLDENS.items() if "error" not in g])
def test_oracle_matches_goldens(name):
    g = GOLDENS[name]
    conf, st = conf_state(synth.Progen3Arch(**g["arch"]), g["seed"])
    ids = sorted(g["records"])
    ll, ppl = O.score(st, conf, [g["records"][i] for i in ids])
    want = pd.read_csv(io.StringIO(g["csv"]))
    assert list(want["sequence_id"]) == ids
    # fp64 against the reference's fp32: measured <= 6.1e-7 over the goldens
    assert np.abs(ll - want["log_likelihood"].to_numpy()).max() < 5e-6
    assert np.abs(ppl / want["perplexity"].to_numpy() - 1).max() < 5e-6


def test_dense_all_experts_golden_is_the_reference_failure():
    assert "einsum" in GOLDENS["dense_all_experts"]["error"]


def test_encoding_of_both_directions():
    tok = Progen3Tokenizer()
    assert tok.encode("ACD") == [1, 6, 8, 10, 11, 7, 2]
    assert tok.encode("ACD", reverse=True) == [1, 7, 11, 10, 8, 6, 2]
    assert tok.encode("ACBJOUXZ") == [1, 6, 8, 10, 9, 17, 22, 28, 31, 33, 7, 2]
    assert tok.encode("acdGH*-") == [1, 6, 14, 15, 7, 2]   # bytes outside the vocabulary are dropped
    assert tok.encode("") == [1, 6, 7, 2]
    with pytest.raises(NotImplementedError):
        tok.encode("AC<eos>D")


def test_fasta_reader(tmp_path):
    p = tmp_path / "x.fasta"
    p.write_text("junk before\n>b desc here\nACD\nEF \n\n>a\r\nGG\r\n>\nKK\n>b\nMM\n")
    assert read_fasta(str(p)) == {"b": "MM", "a": "GG", "": "KK"}


def test_config_parsing_and_refusals():
    base = synth.Progen3Arch(2, 256, 4, 2, 512).config()
    c = checkpoint.progen3_config(base)
    assert (c.kv_heads, c.n_experts, c.top_k, c.vocab, c.rope_theta) == (2, 8, 2, 134, 1e5)
    assert checkpoint.progen3_config({**base, "intermediate_size": None, "gated_mlp": True}).ffn_dim == 3 * 256
    assert checkpoint.progen3_config({**base, "num_experts_per_tok": 9}).top_k == 8
    assert checkpoint.progen3_config({**base, "num_key_value_heads": None}).kv_heads == 4
    with pytest.raises(NotImplementedError, match="silu"):
        checkpoint.progen3_config({**base, "hidden_act": "gelu"})
    with pytest.raises(NotImplementedError, match="clip_qkv"):
        checkpoint.progen3_config({**base, "clip_qkv": 8.0})
    with pytest.raises(NotImplementedError, match="head_dim"):
        checkpoint.progen3_config({**base, "num_attention_heads": 8})
    with pytest.raises(ValueError, match="num_key_value_heads"):
        checkpoint.progen3_config({**base, "num_key_value_heads": 3})
    with pytest.raises(NotImplementedError, match="GB in fp32"):
        checkpoint.progen3_config({})  # the 46B defaults


@pytest.mark.parametrize("field,value,msg", [("heads", 6, "head_dim"), ("kv_heads", 3, "num_key_value_heads"),
                                              ("top_k", 9, "num_experts_per_tok"), ("n_experts", 65, "num_experts")])
def test_pg_create_refusals(field, value, msg):
    lib = _lib.load()
    desc = _lib.PgModelDesc(arch=_lib.PG_ARCH_PROGEN3, layers=2, embed_dim=1024, heads=16, ffn_dim=512, vocab=134, max_positions=64,
                            precision=_lib.PG_PREC_F16F8, kv_heads=4, n_experts=8, top_k=2, rms_eps=1e-5)
    setattr(desc, field, value)
    h = C.c_void_p()
    assert lib.pg_create(C.byref(desc), C.byref(h)) == 4  # PG_ERR_UNSUPPORTED, before any device is touched
    assert msg in lib.pg_last_error(None).decode()


@pytest.mark.parametrize("gated", [False, True])
def test_megablocks_and_eager_layouts_give_the_same_oracle_logits(gated):
    arch = synth.Progen3Arch(2, 256, 4, 2, 256, gated_mlp=gated)
    st = synth.make_progen3_state(arch, 7)
    conf = checkpoint.progen3_config(arch.config())
    eager = checkpoint.normalise_progen3_state(conf, st)
    mb = checkpoint.normalise_progen3_state(conf, synth.progen3_megablocks_state(arch, st))
    fused = checkpoint.normalise_progen3_state(conf, {k.replace(".self_attn.", ".norm_attn_norm.self_attn."): v for k, v in st.items()})
    ids = Progen3Tokenizer().encode("MKVLAAGICW")
    want, _ = O.forward(eager, conf, ids)
    for other in (mb, fused):
        assert sorted(other) == sorted(eager)
        got, _ = O.forward(other, conf, ids)
        assert torch.equal(got, want)


def test_cli_flags_match_the_reference():
    from proteingym_b200 import score_progen3
    ref = json.load(open(os.path.join(GOLDEN, "progen3_cli_flags.json")))["options"]
    acts = {a.dest: a for a in score_progen3.create_parser()._actions}
    for o in ref:
        a = acts[o["name"]]
        assert a.option_strings == o["opts"] and a.required == o["required"]
        if not o["required"]:
            assert a.default == (False if o["is_flag"] else o["default"])
        assert (a.nargs == 0) == o["is_flag"]


def test_product_path_never_imports_the_oracle():
    code = ("import sys; sys.path.insert(0, %r); import proteingym_b200.score_progen3, proteingym_b200.progen3_engine, "
            "proteingym_b200.checkpoint; print(any(m == 'oracle' or m.startswith('oracle.') for m in sys.modules))" % ROOT)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True).stdout.strip()
    assert out == "False"
