"""CPU: RITA host logic against the goldens of the unmodified reference (oracle/gen_golden_rita.py): the fp32 oracle reproduces the
reference's scores, the tokenizer matches the ``tokenizers`` library on both fixture files, the chunk plan and its NaN / failure edges,
row de-duplication and the prefix plan, the drop-in CLI's flags, the checkpoint loader's key mapping and tying rule, and refusals."""
import json
import os
import re
import warnings

import numpy as np
import pandas as pd
import pytest
import torch

from oracle import rita_oracle as O
from proteingym_b200 import checkpoint, synth
from proteingym_b200.rita_engine import RitaTokenizer, chunks, plan
from proteingym_b200.tranception_engine import apply_substitutions, prefix_split

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN_OK = ["tiny", "tiny_bos", "tiny_untied", "indels", "long_1100", "long_2047", "long_2046_bos"]  # true sizes: test_gpu_rita.py


def load_golden(name):
    with open(os.path.join(GOLDEN, f"rita_{name}_meta.json")) as fh:
        meta = json.load(fh)
    a = meta["arch"]
    arch = synth.RitaArch(a["layers"], a["embed_dim"], a["heads"], a["ff_ratio"], a["vocab"])
    dms = pd.read_csv(os.path.join(GOLDEN, f"rita_{name}_dms.csv"))
    if meta["indel_mode"]:
        seqs = list(dms["mutated_sequence"])
    else:
        seqs = [apply_substitutions(meta["sequence"], m) for m in dms["mutant"]]
    tok = RitaTokenizer(os.path.join(GOLDEN, f"rita_tokenizer_{meta['tokenizer']}"))
    return meta, arch, seqs, tok


@pytest.mark.parametrize("name", GOLDEN_OK)
def test_oracle_reproduces_reference_golden(name):
    meta, arch, seqs, tok = load_golden(name)
    want = pd.read_csv(os.path.join(GOLDEN, f"rita_{name}_reference_output.csv"))["RITA_score"].to_numpy()
    st = synth.make_rita_state(arch, meta["seed"], meta["untied"])
    got = O.calc_fitness(st, seqs, tok.encode, arch.heads, torch.float32, tied=not meta["untied"])
    assert np.array_equal(np.isnan(got), np.isnan(want))
    if np.isfinite(want).any():
        assert np.nanmax(np.abs(got - want)) <= 2e-5
    if name == "long_2047":
        assert np.isnan(want).all()


@pytest.mark.parametrize("variant", ["plain", "bos_eos"])
def test_tokenizer_matches_tokenizers_library(variant):
    from tokenizers import Tokenizer
    folder = os.path.join(GOLDEN, f"rita_tokenizer_{variant}")
    lib = Tokenizer.from_file(os.path.join(folder, "tokenizer.json"))
    tok = RitaTokenizer(folder)
    rng = np.random.RandomState(1)
    for s in ["", "A", "MKV", "ACDEFGHIKLMNPQRSTVWYXU", "XBZJO*-ak", synth.random_protein(500, 2)] + \
             ["".join(rng.choice(list("ACDXZBUO"), size=n)) for n in (1, 7, 64)]:
        assert tok.encode(s) == lib.encode(s).ids, s
    assert tok.n_special == (2 if variant == "bos_eos" else 0)


def test_tokenizer_refuses_what_it_does_not_implement(tmp_path):
    src = json.load(open(os.path.join(GOLDEN, "rita_tokenizer_plain", "tokenizer.json")))
    for key, val, msg in [("normalizer", {"type": "Lowercase"}, "normalizer"), ("pre_tokenizer", {"type": "Whitespace"}, "pre-tokenizer"),
                          ("post_processor", {"type": "ByteLevel"}, "post-processor")]:
        bad = dict(src, **{key: val})
        p = tmp_path / f"{key}.json"
        p.write_text(json.dumps(bad))
        with pytest.raises(NotImplementedError, match=msg):
            RitaTokenizer(str(p))
    bad = json.loads(json.dumps(src))
    bad["model"]["merges"] = [["A", "C"]]
    (tmp_path / "merges.json").write_text(json.dumps(bad))
    with pytest.raises(NotImplementedError, match="merges"):
        RitaTokenizer(str(tmp_path / "merges.json"))
    bad["model"] = {"type": "WordPiece", "vocab": {}}
    (tmp_path / "wp.json").write_text(json.dumps(bad))
    with pytest.raises(NotImplementedError, match="WordPiece"):
        RitaTokenizer(str(tmp_path / "wp.json"))
    with pytest.raises(NotImplementedError, match="special token"):
        RitaTokenizer(os.path.join(GOLDEN, "rita_tokenizer_plain")).encode("AC<EOS>D")


@pytest.mark.parametrize("L", [1, 1022, 1023, 1024, 1100, 2045, 2046, 2047, 3070])
def test_chunk_plan_and_nan_edges(L):
    p = synth.random_protein(L, 3)
    cs = chunks(p)
    assert "".join(cs) == p
    if L < 1023:
        assert cs == [p]
    else:
        assert len(cs) == 1 + L // 1023 and all(len(c) == 1023 for c in cs[:-1])
    plain = RitaTokenizer(os.path.join(GOLDEN, "rita_tokenizer_plain"))
    bos = RitaTokenizer(os.path.join(GOLDEN, "rita_tokenizer_bos_eos"))
    last = cs[-1]
    # targets per (chunk, direction): no template -> NaN for a one-residue chunk, failure for an empty one; with <BOS>/<EOS> always finite
    assert (len(plain.encode(last)) - 1 <= 0) == (L % 1023 in (0, 1) if L >= 1023 else L <= 1)
    assert (len(plain.encode(last)) == 0) == (L >= 1023 and L % 1023 == 0)
    assert len(bos.encode(last)) - 1 >= 1


def test_dedupe_and_prefix_plan_reconstruct_reference_strings():
    wt = synth.random_protein(1100, 4)
    muts = synth.sample_mutants(wt, 40, 5, multi_frac=0.3, max_sites=3) + [f"{wt[0]}1{'C' if wt[0] != 'C' else 'A'}"]
    prots = [synth.apply_mutant(wt, m) for m in muts] + [wt, wt[:500] + wt[501:]]
    rows, index, wt_of = plan(prots, wt)
    assert len(rows) == len(set(rows))
    for p, idx in zip(prots, index):
        want = [s for c in chunks(p) for s in (c, c[::-1])]
        assert [rows[r] for r in idx] == want  # every planned string is the reference's string, in its summation order
    # a chunk without a mutation is the wild type's row, computed once: the WT's second-chunk rows serve every protein that is unchanged there
    wt_idx = index[prots.index(wt)]
    shared = sum(idx[2:] == wt_idx[2:] for idx in index)
    assert shared == sum(p[1023:] == wt[1023:] for p in prots) >= 20
    assert len({r for idx in index for r in idx}) < 4 * len(prots)
    wt_strings = {(k, dr): s for k, c in enumerate(chunks(wt)) for dr, s in enumerate((c, c[::-1]))}
    tok = RitaTokenizer(os.path.join(GOLDEN, "rita_tokenizer_bos_eos"))
    for r, w in wt_of.items():
        assert rows[w] in wt_strings.values() and len(rows[w]) == len(rows[r]) and rows[w] != rows[r]
        x, y = tok.encode(rows[r]), tok.encode(rows[w])
        fd, start = prefix_split(x, y, 0, 128)
        assert x[:fd] == y[:fd] and x[fd] != y[fd] and start <= fd and start % 128 == 0
        # L->R rows share their prefix up to the first change, R->L rows up to the last change (of the protein)
        k = [i for i, (a, b) in enumerate(zip(rows[r], rows[w])) if a != b]
        assert fd == len(tok.prefix) + k[0]


def test_prefix_split_is_the_tranception_arithmetic():
    # [CLS] offset 1 (Tranception) and token lists without offset (RITA) give the same first-difference token and tile-aligned start
    x, w = "A" * 300 + "C" + "A" * 10, "A" * 311
    assert prefix_split(x, w, 1, 128) == (301, 256)
    assert prefix_split([1] + list(x), [1] + list(w), 0, 128) == (301, 256)
    assert prefix_split(w, w, 1, 128) == (312, 256)


def test_cli_flags_match_reference():
    from proteingym_b200 import score_rita
    with open(os.path.join(GOLDEN, "rita_cli_flags.json")) as fh:
        ref = json.load(fh)
    acts = {a.option_strings[0]: a for a in score_rita.create_parser()._actions if a.dest != "help"}
    for flag, r in ref.items():
        a = acts[flag]
        assert (a.dest, a.default, a.required, getattr(a.type, "__name__", None), a.nargs == 0) == \
               (r["dest"], r["default"], r["required"], r["type"], r["store_true"]), flag
    assert set(acts) - set(ref) == {"--RITA_tokenizer_path", "--precision", "--device"}
    for name in ("tiny", "indels"):
        with open(os.path.join(GOLDEN, f"rita_{name}_meta.json")) as fh:
            assert set(json.load(fh)["argv_flags"]) <= set(ref)


def test_loader_key_mapping_and_tying(tmp_path):
    arch = synth.RitaArch(2, 128, 2)
    st = synth.write_rita_checkpoint(str(tmp_path / "tied"), arch, seed=3)
    conf, state, inv = checkpoint.load_rita_checkpoint(str(tmp_path / "tied"))
    assert (conf.layers, conf.embed_dim, conf.heads, conf.ffn_dim, conf.vocab, conf.tied) == (2, 128, 2, 512, 26, True)
    assert "lm_head.weight" not in state and not any("inv_freq" in k or k.startswith("transformer.") for k in state)
    assert torch.equal(state["layers.1.self_attention.query.weight"], st["transformer.layers.1.self_attention.query.weight"])
    assert torch.equal(inv, st["transformer.layers.0.self_attention.rotary_embedding.inv_freq"])
    cos, sin = checkpoint.rotary_tables(inv, 5)
    assert cos.shape == (5, 32) and torch.equal(cos[3], torch.cos(3 * inv))
    # untied, from safetensors
    synth.write_rita_checkpoint(str(tmp_path / "untied"), arch, seed=3, untied=True, safetensors=True)
    conf, state, _ = checkpoint.load_rita_checkpoint(str(tmp_path / "untied"))
    assert not conf.tied and state["lm_head.weight"].shape == (26, 128)
    # tie_word_embeddings absent + a differing lm_head: tied, with a warning
    cfgp = tmp_path / "untied" / "config.json"
    cfg = json.load(open(cfgp))
    del cfg["tie_word_embeddings"]
    cfgp.write_text(json.dumps(cfg))
    with pytest.warns(UserWarning, match="discarded"):
        conf, state, _ = checkpoint.load_rita_checkpoint(str(tmp_path / "untied"))
    assert conf.tied and "lm_head.weight" not in state
    # layers that disagree on inv_freq, a missing key
    bad = dict(st)
    bad["transformer.layers.1.self_attention.rotary_embedding.inv_freq"] = bad["transformer.layers.1.self_attention.rotary_embedding.inv_freq"] * 2
    synth.write_rita_checkpoint(str(tmp_path / "bad"), arch, state=bad)
    with pytest.raises(ValueError, match="disagree"):
        checkpoint.load_rita_checkpoint(str(tmp_path / "bad"))
    bad = dict(st)
    del bad["transformer.layers.0.mlp.2.bias"]
    synth.write_rita_checkpoint(str(tmp_path / "bad2"), arch, state=bad)
    with pytest.raises(ValueError, match="mlp.2.bias"):
        checkpoint.load_rita_checkpoint(str(tmp_path / "bad2"))


def test_refusals_are_in_the_library_and_its_architecture_table():
    src = open(os.path.join(os.path.dirname(GOLDEN), "..", "proteingym_b200", "csrc", "api.cu")).read()
    assert "RITA needs head_dim 64" in src and "has no retrieval fusion" in src
    assert re.search(r'\{PG_ARCH_RITA,\s*"RITA",\s*FAM_DECODER,\s*false,', src)  # no retrieval fusion
    hdr = open(os.path.join(os.path.dirname(GOLDEN), "..", "include", "pgscore.h")).read()
    assert "PG_ARCH_RITA = 5" in hdr

