"""ORACLE SUPPORT — regenerates the ProGen2 goldens by running the UNMODIFIED ProGen2 compute_fitness.py ``main()`` (reference root
proteingym/baselines/progen2) on the CPU, through oracle/ref_shims_progen2.py, on seeded synthetic ProGen2 weights
(synth.make_progen2_state). Everything goes to one JSON-lines file, tests/golden/progen2_goldens.jsonl: per case one ``"kind": "case"``
line (seed, arch, target sequence, mode, CPU seconds, the DMS input as columns, and the Progen2_score column of the reference's output CSV,
whose other columns are the DMS file's mutant and DMS_score, or the exception it raised); the reference argparse surface (``"cli_flags"``);
and the reference tokenizer's encodings of tricky strings (``"encoding"``). Regenerated entries replace their old lines.
Usage: python oracle/gen_golden_progen2.py [case ... | flags | tokenizer]"""
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
from oracle import ref_shims_progen2 as R  # noqa: E402
from proteingym_b200 import synth  # noqa: E402

GOLDEN_FILE = os.path.join(ROOT, "tests", "golden", "progen2_goldens.jsonl")
AA = synth.AA20
TINY = synth.Progen2Arch(2, 512, 8, 32)             # head_dim 64, rotary_dim = hd / 2
TINY_R16 = synth.Progen2Arch(2, 512, 8, 16)         # rotary_dim < hd / 2
TINY_96 = synth.Progen2Arch(2, 768, 8, 96)          # head_dim 96, the whole head rotated
TINY_NONE = synth.Progen2Arch(2, 512, 8, None)      # rotary_dim null: ProGenModel.__init__ fails on it (modeling_progen.py:325)
TINY_80 = synth.Progen2Arch(2, 640, 8, 64)          # head_dim 80, rotary_dim 64
TINY_2K = synth.Progen2Arch(2, 512, 8, 32, 2048)


def _sub(seq, p, k=3):
    return f"{seq[p]}{p + 1}{AA[(AA.index(seq[p]) + k) % 20]}"


# name -> arch, protein length, mutants (n sampled, multi-mutant fraction, extra sites), mode, seed.
# mode "wrap": no mutated_sequence column (the reference builds "1" + seq + "2"); "column": the column holds the raw mutated sequences;
# "indels": --indel_mode on random indels; "raw": the column holds the given strings (`seqs`).
CASES = {
    "tiny_wrap": dict(arch=TINY, L=150, n=40, multi=0.3, seed=31, mode="wrap"),
    "tiny_column": dict(arch=TINY, L=150, n=40, multi=0.3, seed=32, mode="column"),
    "tiny_rejected": dict(arch=TINY, L=40, n=5, seed=33, mode="wrap", bad="A3C"),
    "indels": dict(arch=TINY, L=140, n=30, seed=34, mode="indels"),
    "rot16": dict(arch=TINY_R16, L=200, n=16, multi=0.2, seed=35, mode="column", sites=[5, 130, 199]),
    "hd96_full_rotary": dict(arch=TINY_96, L=300, n=16, multi=0.2, seed=36, mode="wrap", sites=[0, 127, 128, 299]),
    "hd80": dict(arch=TINY_80, L=300, n=16, multi=0.2, seed=37, mode="column", sites=[0, 129, 257, 299]),
    "rotary_none": dict(arch=TINY_NONE, L=60, n=4, seed=53, mode="column"),
    "dropped_chars": dict(arch=TINY, seed=38, mode="raw", L=60,
                          seqs=["mkvACDEFGHIK", "ACJDEFGH-IKL", "AC DE\tFG*HI", "ACDEFGHIKLMNPQRSTVWYBXZOU", "1ACDEFGHIK2"]),
    "terminal_inside": dict(arch=TINY, seed=39, mode="raw", L=60, seqs=["ACDEFGHIK", "ACD1EFGHIK"]),  # the reference asserts
    "long_1023": dict(arch=TINY, L=1023, n=6, seed=40, mode="column", sites=[0, 1022]),
    "long_1024": dict(arch=TINY, L=1024, n=4, seed=41, mode="column", sites=[0, 1023]),      # empty last chunk: fails
    "long_1025": dict(arch=TINY, L=1025, n=4, seed=42, mode="column", sites=[0, 1024]),      # 1-character chunk: fails
    "long_1026": dict(arch=TINY, L=1026, n=6, seed=43, mode="column", sites=[0, 1023, 1024, 1025]),
    "long_2048": dict(arch=TINY, L=2048, n=4, seed=44, mode="column", sites=[0, 2047]),      # empty last chunk: fails
    "long_2049": dict(arch=TINY, L=2049, n=4, seed=45, mode="column", sites=[0, 2048]),      # 1-character chunk: fails
    "long_2053": dict(arch=TINY, L=2053, n=6, seed=46, mode="column", sites=[0, 1100, 2050]),
    "wrap_1022": dict(arch=TINY, L=1022, n=4, seed=47, mode="wrap", sites=[0, 1021]),        # "1" + 1022 + "2" = 1024: fails
    "wrap_1024": dict(arch=TINY, L=1024, n=6, seed=48, mode="wrap", sites=[0, 500, 1023]),   # last chunk "X2": NaN
    "ctx2k_2047": dict(arch=TINY_2K, L=2047, n=6, seed=49, mode="column", sites=[0, 1500, 2046]),
    "ctx2k_2049": dict(arch=TINY_2K, L=2049, n=4, seed=50, mode="column", sites=[0, 2048]),  # 1-character chunk: fails
    "ctx2k_2050": dict(arch=TINY_2K, L=2050, n=6, seed=51, mode="column", sites=[0, 2047, 2049]),
    "ctx2k_4097": dict(arch=TINY_2K, L=4097, n=2, seed=52, mode="column", sites=[4096]),      # 1-character chunk: fails
    "progen2_small": dict(arch=synth.PROGEN2_SMALL, L=300, n=10, multi=0.2, seed=61, mode="wrap", sites=[10, 130, 250], true_size=True),
    "progen2_medium": dict(arch=synth.PROGEN2_MEDIUM, L=300, n=10, multi=0.2, seed=62, mode="column", sites=[10, 130, 250], true_size=True),
    "progen2_large": dict(arch=synth.PROGEN2_LARGE, L=260, n=10, multi=0.2, seed=63, mode="wrap", sites=[10, 130, 250], true_size=True),
}
TRICKY = ["", "A", "1MKVA2", "2AC1", "mkv", "AC-D", "ACJ D", "ACDEFGHIKLMNPQRSTVWY", "BOUXZ", "J", "aA", " A", "A\n", "Ä",
          "ÅCD", "12", "1", "2", "3A4", "A*C", "acdefghiklmnpqrstvwyBXZ", "<A>", "MKV|L", "é1Z"]


def case_dms(c):
    seq = synth.random_protein(c["L"], c["seed"])
    rng = np.random.RandomState(c["seed"])
    if c["mode"] == "raw":
        df = pd.DataFrame({"mutant": [f"seq{i}" for i in range(len(c["seqs"]))], "mutated_sequence": c["seqs"]})
    elif c["mode"] == "indels":
        ms = synth.random_indels(seq, c["n"], c["seed"])
        df = pd.DataFrame({"mutant": [f"indel{i}" for i in range(len(ms))], "mutated_sequence": ms})
    else:
        muts = synth.sample_mutants(seq, c["n"], c["seed"], multi_frac=c.get("multi", 0.0), max_sites=3)
        muts += [_sub(seq, p) for p in c.get("sites", [])]
        if c.get("bad"):
            muts.append(c["bad"] if seq[2] != c["bad"][0] else "W3C")
        df = pd.DataFrame({"mutant": muts})
        if c["mode"] == "column":
            df["mutated_sequence"] = [synth.apply_mutant(seq, m) for m in muts]
    df["DMS_score"] = rng.randn(len(df))
    return seq, df


def run_case(name, cf):
    c = CASES[name]
    seq, df = case_dms(c)
    a = c["arch"]
    meta = dict(kind="case", name=name, arch=dataclasses.asdict(a), seed=c["seed"], mode=c["mode"], indel_mode=c["mode"] == "indels", sequence=seq,
                true_size=bool(c.get("true_size")))
    if c.get("true_size"):
        meta["assumed"] = ("the released config.json files are not available here: layers, width, heads, rotary_dim and n_positions "
                           "are the commonly published values (synth.PROGEN2_*); the weights are seeded random draws")
    with tempfile.TemporaryDirectory() as tmp:
        model = os.path.join(tmp, "model")
        synth.write_progen2_checkpoint(model, a, seed=c["seed"])
        os.makedirs(os.path.join(tmp, "dms"))
        df.to_csv(os.path.join(tmp, "dms", "ASSAY.csv"), index=False)
        pd.DataFrame({"DMS_id": ["ASSAY"], "DMS_filename": ["ASSAY.csv"], "target_seq": [seq]}).to_csv(os.path.join(tmp, "ref.csv"), index=False)
        os.makedirs(os.path.join(tmp, "out"))
        argv = ["compute_fitness.py", "--Progen2_model_name_or_path", model, "--DMS_reference_file_path", os.path.join(tmp, "ref.csv"),
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
    meta["argv_flags"] = [x for x in argv[1:] if x.startswith("--")]
    meta["dms"] = {c: df[c].tolist() for c in df.columns}
    meta["reference_scores"] = None
    if out is not None:
        assert list(out.columns) == ["mutant", "Progen2_score", "DMS_score"] and out["mutant"].tolist() == df["mutant"].tolist()
        meta["reference_scores"] = out["Progen2_score"].tolist()
        print(name, len(out), "rows,", int(out["Progen2_score"].isna().sum()), "NaN,", meta["cpu_seconds"], "s", flush=True)
    else:
        print(name, "reference raised", meta["error"], flush=True)
    return [meta]


def cli_flags():
    """The reference parser's options (compute_fitness.py:116-125), captured by running its __main__ block up to parse_args."""
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
    return [dict(kind="cli_flags", flags=got)]


def tokenizer_encodings():
    """The reference tokenizer (tokenizer.json beside compute_fitness.py, read as create_tokenizer_custom does) on TRICKY strings."""
    from tokenizers import Tokenizer
    with open(os.path.join(R.REF, "tokenizer.json")) as fh:
        tok = Tokenizer.from_str(fh.read())
    rng = np.random.RandomState(5)
    strings = TRICKY + ["".join(rng.choice(list("ACDEFGHIKLMNPQRSTVWYBJOUXZacgt-*12 "), size=n)) for n in (5, 40, 300)]
    return [dict(kind="encoding", text=s, ids=tok.encode(s).ids) for s in strings]


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    names = sys.argv[1:] or [n for n in CASES if not CASES[n].get("true_size")] + ["flags", "tokenizer"]
    cf = R.install()
    old = [json.loads(x) for x in open(GOLDEN_FILE)] if os.path.exists(GOLDEN_FILE) else []
    key = lambda r: r["name"] if r["kind"] == "case" else r["kind"]  # noqa: E731
    new = {}
    for n in names:
        recs = cli_flags() if n == "flags" else tokenizer_encodings() if n == "tokenizer" else run_case(n, cf)
        new[key(recs[0])] = recs
    order = list(CASES) + ["cli_flags", "encoding"]
    groups = {}
    for r in old:
        groups.setdefault(key(r), []).append(r)
    groups.update(new)
    with open(GOLDEN_FILE, "w") as fh:
        for k in sorted(groups, key=order.index):
            for r in groups[k]:
                fh.write(json.dumps(r, ensure_ascii=False) + "\n")
