"""ORACLE SUPPORT — regenerates tests/golden/rita_* by running the UNMODIFIED RITA compute_fitness.py ``main()`` (reference root
proteingym/baselines/rita) on the CPU, through oracle/ref_shims_rita.py, on seeded synthetic RITA weights (synth.make_rita_state) and the
two synthetic tokenizer files (synth.write_rita_tokenizer: no template, and <BOS> seq <EOS>), which are committed with the goldens.
Per case: the DMS input (``rita_<case>_dms.csv``), the reference's output CSV (``rita_<case>_reference_output.csv``, or the exception
it raised) and a meta file (seed, arch, tokenizer variant, target sequence, CPU seconds); plus the reference argparse surface as
rita_cli_flags.json.  Usage: python oracle/gen_golden_rita.py [case ...]"""
from __future__ import annotations

import argparse
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
from oracle import ref_shims_rita as R  # noqa: E402
from proteingym_b200 import synth  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
TINY = synth.RitaArch(2, 128, 2)
AA = synth.AA20
TOKENIZERS = {"plain": os.path.join(GOLDEN, "rita_tokenizer_plain"), "bos_eos": os.path.join(GOLDEN, "rita_tokenizer_bos_eos")}


def _sub(seq, p, k=3):
    return f"{seq[p]}{p + 1}{AA[(AA.index(seq[p]) + k) % 20]}"


def _arch_name(a):
    return {synth.RITA_S: "RITA_S", synth.RITA_M: "RITA_M", synth.RITA_L: "RITA_L"}.get(a)


# name -> arch, tokenizer variant, protein length, mutants (n sampled, multi-mutant fraction, extra sites), indels, untied head, seed
CASES = {
    "tiny": dict(arch=TINY, tok="plain", L=150, n=60, multi=0.3, seed=11),
    "tiny_bos": dict(arch=TINY, tok="bos_eos", L=150, n=60, multi=0.3, seed=12),
    "tiny_untied": dict(arch=TINY, tok="plain", L=150, n=40, multi=0.2, seed=13, untied=True),
    "tiny_rejected": dict(arch=TINY, tok="plain", L=40, n=5, multi=0.0, seed=14, bad="A3C"),
    "indels": dict(arch=TINY, tok="plain", L=140, n=40, seed=15, indels=True),
    "long_1100": dict(arch=TINY, tok="plain", L=1100, n=12, multi=0.2, seed=16, sites=[0, 1021, 1022, 1023, 1024, 1099]),
    "long_2046": dict(arch=TINY, tok="plain", L=2046, n=8, multi=0.0, seed=17, sites=[0, 1022, 1023, 2045]),  # empty 3rd chunk: raises
    "long_2047": dict(arch=TINY, tok="plain", L=2047, n=8, multi=0.0, seed=18, sites=[0, 1022, 1023, 2046]),  # 1-residue chunk: NaN
    "long_2046_bos": dict(arch=TINY, tok="bos_eos", L=2046, n=8, multi=0.0, seed=17, sites=[0, 1022, 1023, 2045]),
    "rita_s": dict(arch=synth.RITA_S, tok="plain", L=250, n=24, multi=0.2, seed=21, sites=[10, 127, 128, 200]),
    "rita_l": dict(arch=synth.RITA_L, tok="plain", L=250, n=12, multi=0.2, seed=23, sites=[10, 130, 249]),
}


def case_dms(c):
    seq = synth.random_protein(c["L"], c["seed"])
    rng = np.random.RandomState(c["seed"])
    if c.get("indels"):
        ms = [x for x in synth.random_indels(seq, c["n"], c["seed"])]
        df = pd.DataFrame({"mutant": [f"indel{i}" for i in range(len(ms))], "mutated_sequence": ms})
    else:
        muts = synth.sample_mutants(seq, c["n"], c["seed"], multi_frac=c.get("multi", 0.0), max_sites=3)
        muts += [_sub(seq, p) for p in c.get("sites", [])]
        if c.get("bad"):
            muts.append(c["bad"] if seq[2] != c["bad"][0] else "W3C")
        df = pd.DataFrame({"mutant": muts})
    df["DMS_score"] = rng.randn(len(df))
    return seq, df


def run_case(name, cf):
    c = CASES[name]
    seq, df = case_dms(c)
    R.TOKENIZER_DIR = TOKENIZERS[c["tok"]]
    a = c["arch"]
    meta = dict(arch=dict(layers=a.layers, embed_dim=a.embed_dim, heads=a.heads, ff_ratio=a.ff_ratio, vocab=a.vocab), arch_name=_arch_name(a),
                seed=c["seed"], tokenizer=c["tok"], untied=bool(c.get("untied")), indel_mode=bool(c.get("indels")), sequence=seq)
    df.to_csv(os.path.join(GOLDEN, f"rita_{name}_dms.csv"), index=False)
    with tempfile.TemporaryDirectory() as tmp:
        model = os.path.join(tmp, "model")
        synth.write_rita_checkpoint(model, a, seed=c["seed"], untied=bool(c.get("untied")))
        os.makedirs(os.path.join(tmp, "dms"))
        df.to_csv(os.path.join(tmp, "dms", "ASSAY.csv"), index=False)
        pd.DataFrame({"DMS_id": ["ASSAY"], "DMS_filename": ["ASSAY.csv"], "target_seq": [seq]}).to_csv(os.path.join(tmp, "ref.csv"), index=False)
        os.makedirs(os.path.join(tmp, "out"))
        argv = ["compute_fitness.py", "--RITA_model_name_or_path", model, "--DMS_reference_file_path", os.path.join(tmp, "ref.csv"),
                "--DMS_data_folder", os.path.join(tmp, "dms"), "--DMS_index", "0", "--output_scores_folder", os.path.join(tmp, "out")]
        if c.get("indels"):
            argv.append("--indel_mode")
        old = sys.argv
        sys.argv = argv
        t0 = time.time()
        try:
            with torch.no_grad():
                cf.main()
            out = pd.read_csv(os.path.join(tmp, "out", "ASSAY.csv"))
            meta["error"] = None
        except (AssertionError, RuntimeError) as e:  # a rejected mutant; an empty chunk with a template-free tokenizer (float ids)
            out = None
            meta["error"] = dict(type=type(e).__name__, message=str(e))
        finally:
            sys.argv = old
        meta["cpu_seconds"] = round(time.time() - t0, 1)
    meta["argv_flags"] = [x for x in argv[1:] if x.startswith("--")]
    with open(os.path.join(GOLDEN, f"rita_{name}_meta.json"), "w") as fh:
        json.dump(meta, fh, indent=1)
    if out is not None:
        out.to_csv(os.path.join(GOLDEN, f"rita_{name}_reference_output.csv"), index=False)
        print(name, len(out), "rows,", int(out["RITA_score"].isna().sum()), "NaN,", meta["cpu_seconds"], "s")
    else:
        print(name, "reference raised", meta["error"])


def cli_flags():
    """The reference parser's options (compute_fitness.py:63-70), captured by running its __main__ block up to parse_args."""
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
    with open(os.path.join(GOLDEN, "rita_cli_flags.json"), "w") as fh:
        json.dump(got, fh, indent=1)


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    for variant, folder in TOKENIZERS.items():
        synth.write_rita_tokenizer(folder, template=(variant == "bos_eos"))
    cf = R.install()
    for n in sys.argv[1:] or list(CASES) + ["flags"]:
        cli_flags() if n == "flags" else run_case(n, cf)
