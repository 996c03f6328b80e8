"""CPU: ProtGPT2 host logic against the goldens of the unmodified reference (oracle/gen_golden_protgpt2.py): the byte-level BPE encoder
against the ``tokenizers`` library on random and tricky strings and from both tokenizer file layouts, its refusals, the scorer's
arithmetic (mean per (chunk, direction), divided by 2 * n_chunks, and the failure edges) with the fp32 oracle standing in for the GPU
rows, the checkpoint loader's key mapping, tying and refusals, and the drop-in CLI's flags."""
import json
import os
import shutil

import numpy as np
import pandas as pd
import pytest
import torch

from oracle import protgpt2_oracle as O
from proteingym_b200 import checkpoint, synth
from proteingym_b200.protgpt2_engine import Protgpt2Scorer, Protgpt2Tokenizer
from proteingym_b200.tranception_engine import apply_substitutions

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOK_DIR = os.path.join(GOLDEN, "protgpt2_tokenizer")
with open(os.path.join(GOLDEN, "protgpt2_goldens.jsonl")) as _fh:
    CASES = {r["name"]: r for r in map(json.loads, _fh)}
AA = "ACDEFGHIKLMNPQRSTVWY"


def _ref():
    from tokenizers import Tokenizer
    return Tokenizer.from_file(os.path.join(TOK_DIR, "tokenizer.json"))


def test_bpe_matches_tokenizers_on_random_and_tricky_strings():
    ref, tok = _ref(), Protgpt2Tokenizer(TOK_DIR)
    rng = np.random.RandomState(3)
    strings = ["", "A", "a", "acdefghiklmnpqrstvwy", AA, "ABCDEFGHIJKLMNOPQRSTUVWXYZ", "AAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAAA", "W" * 700,
               "LLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLLL", "MkVlAx", "BJOUXZ"]
    strings += ["".join(rng.choice(list(AA), size=n)) for n in rng.randint(1, 1024, size=300)]
    strings += ["".join(rng.choice(list(AA + AA.lower() + "BJOUXZ"), size=n)) for n in (2, 17, 333)]
    for s in strings:
        assert tok.encode(s) == ref.encode(s).ids, s[:40]


def test_vocab_and_merges_files_give_the_same_ids(tmp_path):
    for f in ("vocab.json", "merges.txt"):
        shutil.copy(os.path.join(TOK_DIR, f), tmp_path / f)
    a, b = Protgpt2Tokenizer(TOK_DIR), Protgpt2Tokenizer(str(tmp_path))
    rng = np.random.RandomState(4)
    for n in (1, 2, 5, 64, 500, 1023):
        s = "".join(rng.choice(list(AA), size=n))
        assert a.encode(s) == b.encode(s)


@pytest.mark.parametrize("text", [" A", "AC DE", "A1", "12", "A-C", "A*", "Ä", "é", "A\n", "<|endoftext|>", "AC.D"])
def test_refuses_characters_the_pre_tokenizer_would_split(text):
    with pytest.raises(NotImplementedError):
        Protgpt2Tokenizer(TOK_DIR).encode(text)


@pytest.mark.parametrize("edit", [
    lambda s: s.__setitem__("normalizer", {"type": "NFC"}),
    lambda s: s["pre_tokenizer"].__setitem__("add_prefix_space", True),
    lambda s: s.__setitem__("pre_tokenizer", {"type": "Whitespace"}),
    lambda s: s["model"].__setitem__("byte_fallback", True),
    lambda s: s["model"].__setitem__("dropout", 0.1),
    lambda s: s["model"].__setitem__("continuing_subword_prefix", "##"),
    lambda s: s["model"].__setitem__("end_of_word_suffix", "</w>"),
    lambda s: s["model"].__setitem__("ignore_merges", True),
    lambda s: s.__setitem__("post_processor", {"type": "TemplateProcessing", "single": [], "pair": [], "special_tokens": {}}),
    lambda s: s["model"].__setitem__("type", "WordPiece"),
])
def test_refuses_tokenizer_features(tmp_path, edit):
    spec = json.load(open(os.path.join(TOK_DIR, "tokenizer.json")))
    edit(spec)
    with open(tmp_path / "tokenizer.json", "w") as fh:
        json.dump(spec, fh)
    with pytest.raises(NotImplementedError):
        Protgpt2Tokenizer(str(tmp_path))


def test_special_token_text_is_refused(tmp_path):
    spec = json.load(open(os.path.join(TOK_DIR, "tokenizer.json")))
    spec["added_tokens"].append(dict(spec["added_tokens"][0], id=1, content="MKV"))
    with open(tmp_path / "tokenizer.json", "w") as fh:
        json.dump(spec, fh)
    with pytest.raises(NotImplementedError):
        Protgpt2Tokenizer(str(tmp_path)).encode("AMKVL")


def _seqs(meta):
    dms = pd.DataFrame(meta["dms"])
    if "mutated_sequence" in dms.columns:
        return list(dms["mutated_sequence"])
    return [apply_substitutions(meta["sequence"], m) for m in dms["mutant"]]


def _cpu_scorer(meta, st):
    """The real Protgpt2Scorer.score with its GPU row sums replaced by the fp32 oracle (no handle is created)."""
    arch = synth.Protgpt2Arch(**meta["arch"])
    sc = object.__new__(Protgpt2Scorer)
    sc.conf = checkpoint.Protgpt2Config(arch.layers, arch.embed_dim, arch.heads, arch.ffn_dim, arch.vocab, arch.n_positions)
    sc.tok, sc.context = Protgpt2Tokenizer(TOK_DIR), 1023
    sc.row_sums = lambda toks, wt_of, needed: np.array(
        [float(O.token_logprobs(st, t, arch.heads, torch.float32).double().sum()) if r in needed and len(t) > 1 else 0.0
         for r, t in enumerate(toks)])
    return sc


@pytest.mark.parametrize("name", ["tiny_subs", "tiny_column", "indels", "long_1022", "long_1100"])
def test_score_arithmetic_against_reference(name):
    meta = CASES[name]
    st = synth.make_protgpt2_state(synth.Protgpt2Arch(**meta["arch"]), meta["seed"])
    got = _cpu_scorer(meta, st).score(_seqs(meta), wt=meta["sequence"])
    want = np.array([np.nan if x is None else x for x in meta["reference_scores"]], dtype=np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    assert np.abs(got[ok] - want[ok]).max() < 2e-4


@pytest.mark.parametrize("name", ["long_1023", "long_2046", "long_1024", "long_2047", "one_token"])
def test_reference_failures_raise(name):
    """No token (an empty last chunk), or one token (a 1-character last chunk, or a chunk BPE merges into one token): the reference
    fails, and so does the scorer."""
    meta = CASES[name]
    assert meta["error"] is not None and meta["reference_scores"] is None
    sc = _cpu_scorer(meta, None)
    with pytest.raises(ValueError):
        sc.score(_seqs(meta), wt=meta["sequence"])


def test_substitution_column_matches_reference():
    meta = CASES["tiny_subs"]
    assert _seqs(meta) == meta["reference_mutated_sequence"]


def test_loader_key_mapping_tying_and_refusals(tmp_path):
    arch = synth.Protgpt2Arch(2, 128, 2, n_positions=64, vocab=300)
    st = synth.make_protgpt2_state(arch, 1, buffers=True)
    synth.write_protgpt2_checkpoint(str(tmp_path / "bin"), arch, state=st)
    conf, state = checkpoint.load_protgpt2_checkpoint(str(tmp_path / "bin"))
    assert (conf.layers, conf.embed_dim, conf.heads, conf.ffn_dim, conf.vocab, conf.n_positions) == (2, 128, 2, 512, 300, 64)
    assert "lm_head.weight" not in state and not any(k.endswith(".attn.bias") or k.endswith(".attn.masked_bias") for k in state)
    assert state["h.1.attn.c_attn.weight"].shape == (128, 384)  # Conv1D [in, out] kept
    assert torch.equal(state["wte.weight"], st["transformer.wte.weight"])
    st16 = {k: v.half() if v.is_floating_point() else v for k, v in synth.make_protgpt2_state(arch, 1).items()}
    synth.write_protgpt2_checkpoint(str(tmp_path / "st"), arch, state=st16, safetensors=True)
    _, s2 = checkpoint.load_protgpt2_checkpoint(str(tmp_path / "st"))
    assert s2["wte.weight"].dtype == torch.float32 and set(s2) == set(state)
    for extra, exc in [(dict(activation_function="gelu"), NotImplementedError), (dict(layer_norm_epsilon=1e-6), NotImplementedError),
                       (dict(scale_attn_by_inverse_layer_idx=True), NotImplementedError), (dict(n_head=4), NotImplementedError),
                       (dict(tie_word_embeddings=False), NotImplementedError), (dict(n_inner=500), NotImplementedError),
                       (dict(n_layer=3), ValueError)]:
        d = tmp_path / f"bad{len(os.listdir(tmp_path))}"
        synth.write_protgpt2_checkpoint(str(d), arch, state=st, config_extra=extra)
        with pytest.raises(exc):
            checkpoint.load_protgpt2_checkpoint(str(d))
    d = tmp_path / "ffn"  # n_inner other than 4d, but a multiple of 64: the GEMMs take it as given
    a2 = synth.Protgpt2Arch(1, 128, 2, n_positions=64, vocab=300, n_inner=320)
    synth.write_protgpt2_checkpoint(str(d), a2, seed=2)
    assert checkpoint.load_protgpt2_checkpoint(str(d))[0].ffn_dim == 320


def test_cli_flags_match_reference():
    from proteingym_b200 import score_protgpt2
    want = json.load(open(os.path.join(GOLDEN, "protgpt2_cli_flags.json")))
    p = score_protgpt2.create_parser()
    got = {a.option_strings[0]: a for a in p._actions if a.dest != "help"}
    for flag, spec in want.items():
        a = got[flag]
        assert a.dest == spec["dest"] and a.default == spec["default"] and a.required == spec["required"]
        assert getattr(a.type, "__name__", None) == spec["type"]
        assert spec["store_true"] == (a.nargs == 0)
    assert set(got) - set(want) == {"--precision", "--device"}


def test_refusals_are_in_the_library():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = open(os.path.join(root, "proteingym_b200", "csrc", "api.cu")).read()
    assert "ProtGPT2 needs head_dim 64" in src and "ProtGPT2 has no retrieval fusion" in src
