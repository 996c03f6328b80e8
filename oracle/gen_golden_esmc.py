"""ORACLE SUPPORT — regenerates tests/golden/esmc_* by running the UNMODIFIED evoscale compute_fitness.py (reference root
proteingym/baselines/evoscale) on the CPU, through oracle/ref_shims_evoscale.py, on seeded synthetic ESM C weights at true size
(synth.make_esmc_state). Per case it commits the reference CLI's output CSV, the masked rows it computed (log_softmax of
``ESMC.logits`` at the masked token, in scoring order = sorted residue positions) and a meta file; plus the reference argparse surface
as esmc_cli_flags.json.  Usage: python oracle/gen_golden_esmc.py [case ...]"""
from __future__ import annotations

import argparse
import json
import os
import runpy
import sys
import tempfile

import numpy as np
import pandas as pd
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims_evoscale as R  # noqa: E402
from proteingym_b200 import synth  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
AA = "ACDEFGHIKLMNPQRSTVWY"


def _sub(seq, p, k=3):
    return f"{seq[p]}{p + 1}{AA[(AA.index(seq[p]) + k) % 20]}"


def case_mutants(seq, n, seed, sites=None):
    muts = synth.sample_mutants(seq, n, seed, multi_frac=0.15, max_sites=2)
    if sites:
        muts += [_sub(seq, p) for p in sites] + [f"{_sub(seq, sites[0], 5)}:{_sub(seq, sites[-1], 7)}"]
    L = len(seq)
    bad = [f"{AA[(AA.index(seq[2]) + 1) % 20]}3A", f"{seq[0]}0C", f"{seq[0]}{L + 1}C", "WT", f"{_sub(seq, 5)}:x9", f"{seq[7]}8{seq[7]}"]
    return muts + bad


CASES = {
    "esmc_300m": dict(model_type="esmc_300M", arch=synth.ESMC_300M, L=180, n=400, seed=301),
    "esmc_600m": dict(model_type="esmc_600M", arch=synth.ESMC_600M, L=120, n=200, seed=601),
    "esmc_300m_window": dict(model_type="esmc_300M", arch=synth.ESMC_300M, L=1150, n=0, seed=302,
                             sites=[0, 1, 2, 3, 509, 510, 511, 512, 513, 514, 575, 1150 - 513, 1150 - 511, 1150 - 509, 1147, 1148, 1149]),
}


def run_case(name, cf):
    c = CASES[name]
    seq = synth.random_protein(c["L"], c["seed"])
    muts = case_mutants(seq, c["n"], c["seed"], c.get("sites"))
    rows = []
    orig = cf.ESMC.logits

    def logits(self, inp, config):
        out = orig(self, inp, config)
        toks = inp.sequence if inp.sequence.dim() == 1 else inp.sequence[0]
        i = int((toks == 32).nonzero()[0, 0])
        rows.append(torch.log_softmax(out.logits.sequence[0, i].float(), -1).detach().numpy())
        return out
    cf.ESMC.logits = logits
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        wfile = os.path.join(tmp, "data", "weights", f"{c['model_type'].lower()}_2024_12_v0.pth")
        synth.write_esmc_checkpoint(wfile, c["arch"], seed=c["seed"])
        os.makedirs(os.path.join(tmp, "dms"))
        dms = pd.DataFrame({"mutant": muts, "DMS_score": np.random.RandomState(c["seed"]).randn(len(muts))})
        dms.to_csv(os.path.join(tmp, "dms", "ASSAY.csv"), index=False)
        pd.DataFrame({"DMS_id": ["ASSAY"], "target_seq": [seq]}).to_csv(os.path.join(tmp, "ref.csv"), index=False)
        os.chdir(tmp)
        try:
            with torch.no_grad():
                cf.process_assays_from_file("ref.csv", "dms", None, "out", model_type=c["model_type"])
            out = pd.read_csv(os.path.join(tmp, "out", "ASSAY.csv"))
        finally:
            os.chdir(cwd)
            cf.ESMC.logits = orig
    a = c["arch"]
    meta = dict(model_type=c["model_type"], arch=dict(layers=a.layers, embed_dim=a.embed_dim, ffn_dim=a.ffn_dim), seed=c["seed"],
                sequence=seq, score_column=f"{c['model_type']}_score")
    with open(os.path.join(GOLDEN, f"{name}_meta.json"), "w") as fh:
        json.dump(meta, fh, indent=1)
    out.to_csv(os.path.join(GOLDEN, f"{name}_reference_output.csv"), index=False)
    np.save(os.path.join(GOLDEN, f"{name}_reference_table.npy"), np.stack(rows).astype(np.float32))
    print(name, len(rows), "rows,", int(out[meta["score_column"]].isna().sum()), "NaN of", len(out))


def cli_flags():
    """The reference parser's options (compute_fitness.py:743-762), captured by running its __main__ block up to parse_args."""
    got = {}

    def capture(self, *a, **k):
        for act in self._actions:
            if act.dest == "help":
                continue
            got[act.option_strings[0]] = dict(dest=act.dest, default=act.default, required=act.required,
                                              choices=list(act.choices) if act.choices else None,
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
    with open(os.path.join(GOLDEN, "esmc_cli_flags.json"), "w") as fh:
        json.dump(got, fh, indent=1)


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    cf = R.install()
    for n in sys.argv[1:] or list(CASES) + ["flags"]:
        cli_flags() if n == "flags" else run_case(n, cf)
