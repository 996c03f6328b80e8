"""ORACLE SUPPORT — regenerates the ProtGPT2 goldens by running the UNMODIFIED ProtGPT2 compute_fitness.py ``main()`` (reference root
proteingym/baselines/protgpt2) on the CPU, through oracle/ref_shims_protgpt2.py, on seeded synthetic GPT-2 weights
(synth.make_protgpt2_state) and the fixture tokenizer. Writes:
  * tests/golden/protgpt2_tokenizer/: a byte-level BPE trained with ``tokenizers`` on synthetic proteins (2 500 merges), its ids permuted
    across [0, 50257) so that scored tokens land in N tile 0 and in the last, partial N tile of the 50 257-way head (``tokenizer``);
  * tests/golden/protgpt2_goldens.jsonl: per case one line (arch, seed, target sequence, mode, CPU seconds, the DMS input as columns, and
    the ProtGPT2_score column of the reference's output CSV, or the exception it raised);
  * tests/golden/protgpt2_cli_flags.json: the reference argparse surface (``flags``).
Usage: python oracle/gen_golden_protgpt2.py [tokenizer | flags | case ...]"""
from __future__ import annotations

import argparse
import dataclasses
import json
import os
import runpy
import sys
import tempfile
import time

import numpy as np
import pandas as pd
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims_protgpt2 as R  # noqa: E402
from proteingym_b200 import synth  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
GOLDEN_FILE = os.path.join(GOLDEN, "protgpt2_goldens.jsonl")
TOK_DIR = R.FIXTURE_TOKENIZER
AA = synth.AA20
TINY = synth.Protgpt2Arch(2, 128, 2)   # head_dim 64, the full 50 257-way vocabulary
V = 50257


def train_tokenizer():
    """Byte-level BPE (GPT-2's pre-tokenizer and byte alphabet) trained on 4 000 synthetic proteins whose residues follow a skewed
    distribution, so that merges of 2 to ~6 residues exist; ids then permuted across [0, V) with half the single amino-acid letters in
    tile 0 (ids < 128) and half in the last tile (ids >= 50 176); <|endoftext|> is id 0, as in ProtGPT2."""
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers, processors, trainers
    rng = np.random.RandomState(11)
    p = rng.dirichlet(np.full(20, 0.7))
    corpus = ["".join(rng.choice(list(AA), size=rng.randint(50, 400), p=p)) for _ in range(4000)]
    tok = Tokenizer(models.BPE())
    tok.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
    tok.decoder = decoders.ByteLevel()
    tok.post_processor = processors.ByteLevel(trim_offsets=True)
    tok.train_from_iterator(corpus, trainers.BpeTrainer(vocab_size=257 + 2500, initial_alphabet=pre_tokenizers.ByteLevel.alphabet(),
                                                          special_tokens=["<|endoftext|>"], show_progress=False))
    spec = json.loads(tok.to_str())
    vocab = spec["model"]["vocab"]
    names = sorted(vocab, key=lambda t: vocab[t])
    ids = list(rng.choice(np.arange(128, V - 81), size=len(names), replace=False))
    first, last = list(range(1, 128)), list(range(V - 81, V))
    new = {}
    for k, t in enumerate(names):
        if t == "<|endoftext|>":
            new[t] = 0
        elif t in AA:
            new[t] = first.pop(0) if AA.index(t) % 2 == 0 else last.pop()
        else:
            new[t] = int(ids[k])
    # a few frequent merges (the first ones learned) also go to the edge tiles
    merged = [t for t in names if len(t) > 1 and t != "<|endoftext|>"]
    for t in merged[:12]:
        new[t] = first.pop() if len(first) > len(last) else last.pop(0)
    spec["model"]["vocab"] = new
    for a in spec["added_tokens"]:
        a["id"] = new[a["content"]]
    os.makedirs(TOK_DIR, exist_ok=True)
    with open(os.path.join(TOK_DIR, "tokenizer.json"), "w") as fh:
        json.dump(spec, fh, ensure_ascii=False)
    with open(os.path.join(TOK_DIR, "vocab.json"), "w") as fh:
        json.dump(new, fh, ensure_ascii=False)
    with open(os.path.join(TOK_DIR, "merges.txt"), "w", encoding="utf-8") as fh:
        fh.write("#version: 0.2\n")
        for m in spec["model"]["merges"]:
            fh.write((m if isinstance(m, str) else " ".join(m)) + "\n")
    with open(os.path.join(TOK_DIR, "tokenizer_config.json"), "w") as fh:
        json.dump(dict(tokenizer_class="GPT2TokenizerFast", bos_token="<|endoftext|>", eos_token="<|endoftext|>", unk_token="<|endoftext|>",
                       add_prefix_space=False, model_max_length=1024), fh, indent=1)
    check = Tokenizer.from_file(os.path.join(TOK_DIR, "tokenizer.json"))
    print("fixture tokenizer:", len(new), "tokens;", check.encode(corpus[0][:60]).ids[:10])


def one_token_word():
    """A multi-character string of amino acids that the fixture tokenizer encodes as ONE token (forward direction)."""
    from tokenizers import Tokenizer
    tok = Tokenizer.from_file(os.path.join(TOK_DIR, "tokenizer.json"))
    words = sorted((t for t in tok.get_vocab() if t.isalpha() and t.isupper() and len(t) >= 3), key=lambda t: (-len(t), t))
    return next(w for w in words if len(tok.encode(w).ids) == 1)


def _sub(seq, p, k=3):
    return f"{seq[p]}{p + 1}{AA[(AA.index(seq[p]) + k) % 20]}"


# name -> arch, protein length, mutants (n sampled, multi-mutant fraction, extra sites), mode, seed.
# mode "wrap": no mutated_sequence column (the reference builds it); "column": the column holds the mutated sequences; "indels":
# --indel_mode on random indels; "raw": the column holds the given strings.
CASES = {
    "tiny_subs": dict(arch=TINY, L=150, n=40, multi=0.3, seed=71, mode="wrap"),
    "tiny_column": dict(arch=TINY, L=300, n=30, multi=0.2, seed=72, mode="column", sites=[0, 150, 299]),
    "indels": dict(arch=TINY, L=140, n=30, seed=73, mode="indels"),
    "one_token": dict(arch=TINY, L=60, seed=74, mode="raw"),
    "long_1022": dict(arch=TINY, L=1022, n=6, seed=75, mode="column", sites=[0, 600, 1021]),
    "long_1100": dict(arch=TINY, L=1100, n=6, seed=76, mode="column", sites=[0, 1022, 1023, 1099]),
    "long_1024": dict(arch=TINY, L=1024, n=4, seed=77, mode="column", sites=[0, 1023]),      # 1-character last chunk
    "long_2047": dict(arch=TINY, L=2047, n=4, seed=78, mode="column", sites=[0, 1500, 2046]),  # 1-character last chunk
    "long_1023": dict(arch=TINY, L=1023, n=4, seed=79, mode="column", sites=[0, 1022]),      # empty last chunk: the reference fails
    "long_2046": dict(arch=TINY, L=2046, n=4, seed=80, mode="column", sites=[0, 2045]),      # empty last chunk: the reference fails
    "protgpt2_true": dict(arch=synth.PROTGPT2, L=300, n=8, multi=0.2, seed=81, mode="wrap", sites=[10, 150, 290], true_size=True),
}


def case_dms(c):
    seq = synth.random_protein(c["L"], c["seed"])
    rng = np.random.RandomState(c["seed"])
    if c["mode"] == "raw":
        w = one_token_word()
        seqs = [w, seq, w + seq[:20], seq[:30] + w]
        df = pd.DataFrame({"mutant": [f"seq{i}" for i in range(len(seqs))], "mutated_sequence": seqs})
    elif c["mode"] == "indels":
        ms = synth.random_indels(seq, c["n"], c["seed"])
        df = pd.DataFrame({"mutant": [f"indel{i}" for i in range(len(ms))], "mutated_sequence": ms})
    else:
        muts = synth.sample_mutants(seq, c["n"], c["seed"], multi_frac=c.get("multi", 0.0), max_sites=3)
        muts += [_sub(seq, p) for p in c.get("sites", [])]
        df = pd.DataFrame({"mutant": muts})
        if c["mode"] == "column":
            df["mutated_sequence"] = [synth.apply_mutant(seq, m) for m in muts]
    df["DMS_score"] = rng.randn(len(df))
    return seq, df


def run_case(name, cf):
    c = CASES[name]
    seq, df = case_dms(c)
    a = c["arch"]
    meta = dict(kind="case", name=name, arch=dataclasses.asdict(a), seed=c["seed"], mode=c["mode"], indel_mode=c["mode"] == "indels",
                sequence=seq, true_size=bool(c.get("true_size")))
    if c.get("true_size"):
        meta["assumed"] = ("ProtGPT2's published shape (GPT-2 large: 36 layers, 1280 wide, 20 heads, n_positions 1024, vocab 50 257) with "
                           "seeded random weights and the fixture tokenizer")
    with tempfile.TemporaryDirectory() as tmp:
        model = os.path.join(tmp, "model")
        synth.write_protgpt2_checkpoint(model, a, seed=c["seed"])
        os.makedirs(os.path.join(tmp, "dms"))
        df.to_csv(os.path.join(tmp, "dms", "ASSAY.csv"), index=False)
        pd.DataFrame({"DMS_id": ["ASSAY"], "DMS_filename": ["ASSAY.csv"], "target_seq": [seq]}).to_csv(os.path.join(tmp, "ref.csv"), index=False)
        os.makedirs(os.path.join(tmp, "out"))
        argv = ["compute_fitness.py", "--ProtGPT2_model_name_or_path", model, "--DMS_reference_file_path", os.path.join(tmp, "ref.csv"),
                "--DMS_data_folder", os.path.join(tmp, "dms"), "--DMS_index", "0", "--output_scores_folder", os.path.join(tmp, "out")]
        if c["mode"] == "indels":
            argv.append("--indel_mode")
        old = sys.argv
        sys.argv = argv
        t0 = time.time()
        try:
            with torch.no_grad():
                cf.main()
            out = pd.read_csv(os.path.join(tmp, "out", "ASSAY.csv"))
            meta["error"] = None
        except (AssertionError, RuntimeError, IndexError, ValueError, TypeError) as e:
            out = None
            meta["error"] = dict(type=type(e).__name__, message=str(e)[:300])
        finally:
            sys.argv = old
        meta["cpu_seconds"] = round(time.time() - t0, 1)
    meta["dms"] = {k: df[k].tolist() for k in df.columns}
    meta["reference_scores"] = None
    if out is not None:
        assert list(out.columns) == ["mutated_sequence", "ProtGPT2_score", "DMS_score"]
        meta["reference_mutated_sequence"] = out["mutated_sequence"].tolist()
        meta["reference_scores"] = [None if np.isnan(x) else x for x in out["ProtGPT2_score"].tolist()]
        print(name, len(out), "rows,", int(out["ProtGPT2_score"].isna().sum()), "NaN,", meta["cpu_seconds"], "s", flush=True)
    else:
        print(name, "reference raised", meta["error"], flush=True)
    return meta


def cli_flags():
    """The reference parser's options (compute_fitness.py:66-72), captured by running its __main__ block up to parse_args."""
    got = {}

    def capture(self, *a, **k):
        for act in self._actions:
            if act.dest == "help":
                continue
            got[act.option_strings[0]] = dict(dest=act.dest, default=act.default, required=act.required, type=getattr(act.type, "__name__", None),
                                              store_true=isinstance(act, argparse._StoreTrueAction))
        raise SystemExit(0)
    orig = argparse.ArgumentParser.parse_args
    argparse.ArgumentParser.parse_args = capture
    try:
        runpy.run_path(os.path.join(R.REF, "compute_fitness.py"), run_name="__main__")
    except SystemExit:
        pass
    finally:
        argparse.ArgumentParser.parse_args = orig
    with open(os.path.join(GOLDEN, "protgpt2_cli_flags.json"), "w") as fh:
        json.dump(got, fh, indent=1)


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    names = sys.argv[1:] or ["tokenizer", "flags"] + list(CASES)
    if "tokenizer" in names:
        train_tokenizer()
    if "flags" in names:
        cli_flags()
    cases = [n for n in names if n in CASES]
    if cases:
        cf = R.install()
        old = {r["name"]: r for r in map(json.loads, open(GOLDEN_FILE))} if os.path.exists(GOLDEN_FILE) else {}
        for n in cases:
            old[n] = run_case(n, cf)
        with open(GOLDEN_FILE, "w") as fh:
            for n in sorted(old, key=list(CASES).index):
                fh.write(json.dumps(old[n]) + "\n")
