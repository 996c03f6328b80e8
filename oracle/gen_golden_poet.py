"""ORACLE SUPPORT — regenerates the PoET goldens by running the UNMODIFIED PoET scripts/score.py ``main()`` (reference root
proteingym/baselines/PoET) on the CPU in fp32, through oracle/ref_shims_poet.py, on seeded synthetic checkpoints
(synth.write_poet_checkpoint) and synthetic a3m files built from real wild types of reference_files/DMS_substitutions.csv.
Everything goes to one JSON-lines file, tests/golden/poet_goldens.jsonl: per case one ``"kind": "case"`` line with the arch, seed, the
reference-file row, the DMS input, the a3m rows, the flags, the PoET_score column of the reference's output CSV (or the exception it
raised), CPU seconds, and per max_similarity the reference sampler's index list and per (context length, max_similarity) the token
lengths of the sampled context in order (which pins the overshoot and the shuffle). The reference argparse surface goes to
tests/golden/poet_cli_flags.json. Regenerated entries replace their old lines.
Usage: python oracle/gen_golden_poet.py [case ... | flags]"""
from __future__ import annotations

import dataclasses
import json
import os
import sys
import tempfile
import time

import numpy as np
import pandas as pd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims_poet as R  # noqa: E402
from proteingym_b200 import synth  # noqa: E402

GOLDEN_FILE = os.path.join(ROOT, "tests", "golden", "poet_goldens.jsonl")
FLAGS_FILE = os.path.join(ROOT, "tests", "golden", "poet_cli_flags.json")
REF_FILE = os.path.join(os.path.dirname(os.path.dirname(R.REF)), "..", "reference_files", "DMS_substitutions.csv")
SIMS = [1.0, 0.95, 0.90, 0.70, 0.50]
TINY = synth.PoetArch(2, 128, 2)
TINY_NORM = synth.PoetArch(2, 128, 2, norm=True)
TINY_3 = synth.PoetArch(3, 192, 3, ff_dim=320)

# name -> arch, reference-file row, window (MSA_start, MSA_end) within the target (None = whole), variants, MSA rows, flags, seed.
# variants: ("subs", n, multi) single/multi substitutions of the target (full sequences); ("indels", n); ("raw", [strings]).
CASES = {
    "subs": dict(arch=TINY, row=0, window=(3, 60), var=("subs", 24, 0.3), msa=40, ctx=[64, 300], seed=11),
    "subs_norm_relative": dict(arch=TINY_NORM, row=1, window=(1, 70), var=("subs", 16, 0.3), msa=30, ctx=[64, 300], seed=12, relative=True),
    "indels": dict(arch=TINY, row=2, window=(5, 55), var=("indels", 16), msa=30, ctx=[100, 257], seed=13),
    "x_targets": dict(arch=TINY_NORM, row=3, window=(1, 50), var=("raw", ["XX", "AXC", "JBZOU"]), msa=20, ctx=[64], seed=14),
    "gappy_rows": dict(arch=TINY_3, row=4, window=(1, 60), var=("subs", 12, 0.0), msa=25, ctx=[64, 300], seed=15, gappy=True),
    "filters_empty": dict(arch=TINY, row=5, window=(1, 40), var=("subs", 8, 0.0), msa=12, ctx=[64, 200], seed=16, identical=True),
    "long_context": dict(arch=TINY, row=6, window=(1, 90), var=("subs", 10, 0.2), msa=400, ctx=[6144], seed=17),
    "batch_size_3": dict(arch=TINY, row=7, window=(1, 45), var=("subs", 10, 0.2), msa=30, ctx=[64, 300], seed=18, batch_size=3),
    "fail_first_row": dict(arch=TINY, row=8, window=(1, 40), var=("subs", 4, 0.0), msa=10, ctx=[64], seed=19, bad_first=True),
    "fail_gap_variant": dict(arch=TINY, row=9, window=(1, 40), var=("raw", ["AC-DE"]), msa=10, ctx=[64], seed=20),
    "fail_all_gap_row": dict(arch=TINY, row=10, window=(1, 40), var=("subs", 4, 0.0), msa=10, ctx=[64], seed=21, all_gap=True),
    "poet_true_shape": dict(arch=synth.POET, row=11, window=(1, 120), var=("subs", 6, 0.3), msa=40, ctx=[400], seed=22, true_size=True),
}


def reference_row(i: int):
    df = pd.read_csv(REF_FILE)
    return df.iloc[i]


def build_inputs(name: str, c: dict, folder: str):
    ref = reference_row(c["row"])
    target = ref["target_seq"]
    s, e = c["window"]
    e = min(e, len(target))
    wt = target[s - 1:e]
    rng = np.random.RandomState(c["seed"])
    kind = c["var"][0]
    if kind == "subs":
        muts = synth.sample_mutants(wt, c["var"][1], c["seed"], multi_frac=c["var"][2])
        seqs = [synth.apply_mutant(wt, m) for m in muts]
    elif kind == "indels":
        seqs = synth.random_indels(wt, c["var"][1], c["seed"])
    else:
        seqs = list(c["var"][1])
    rows = synth.poet_a3m(wt, c["msa"], c["seed"])
    if c.get("gappy"):
        rows[3] = "A" + "-" * (len(wt) - 1)                           # one residue
        rows[5] = "-" * (len(wt) - 2) + "ww" + wt[-2:]                 # insertions only before the last columns
    if c.get("identical"):
        rows = [wt] * c["msa"]
    if c.get("bad_first"):
        rows[0] = wt[:-1] + ("A" if wt[-1] != "A" else "C")
    if c.get("all_gap"):
        rows[4] = "-" * len(wt)
    dms_file = f"{name}.csv"
    pd.DataFrame({"mutated_sequence": seqs, "DMS_score": rng.randn(len(seqs))}).to_csv(os.path.join(folder, "dms", dms_file), index=False)
    pd.DataFrame([{"DMS_id": name, "DMS_filename": dms_file, "target_seq": target, "MSA_start": s, "MSA_end": e}]).to_csv(
        os.path.join(folder, "ref.csv"), index=False)
    with open(os.path.join(folder, "msa", f"{name}.a3m.zst"), "w") as fh:
        for i, r in enumerate(rows):
            fh.write(f">seq{i}\n{r}\n")
    return dict(DMS_filename=dms_file, target_seq=target, MSA_start=s, MSA_end=e), seqs, rows, wt


def sampler_record(mod, rows, wt, ctx, seed):
    """The reference sampler's index lists per max_similarity and the context token lengths per (context length, max_similarity)."""
    from poet.alphabets import Uniprot21
    from poet.msa.sampling import MSASampler, NeighborsSampler
    alphabet = Uniprot21(include_gap=True, include_startstop=True, distinct_startstop=True)
    seqs = [r.encode() for r in rows]
    try:
        msa = mod.get_encoded_msa_from_a3m_seqs(msa_sequences=seqs, alphabet=alphabet)
        out = {"idxs": {}, "ctx_lens": {}}
        for sim in SIMS:
            idx = MSASampler(method=NeighborsSampler(can_use_torch=False), max_similarity=sim).get_sample_idxs(
                msa=msa, gap_token=alphabet.gap_token, seed=seed)
            out["idxs"][str(sim)] = [int(i) for i in idx]
            for mt in ctx:
                cs = mod.sample_msa_sequences(get_sequence_fn=lambda ii: seqs[ii].upper().translate(None, delete=b"-"), sample_idxs=idx,
                                              max_tokens=mt, alphabet=alphabet, shuffle_seed=seed, truncate=False)
                out["ctx_lens"][f"{mt}:{sim}"] = [int(len(x)) for x in cs]
        return out
    except Exception as e:  # noqa: BLE001 — recorded: the scorer must fail the same way
        return {"error": f"{type(e).__name__}: {e}"}


def run_case(name: str) -> dict:
    c = CASES[name]
    mod = R.install()
    with tempfile.TemporaryDirectory() as tmp:
        for sub in ("dms", "msa", "out"):
            os.makedirs(os.path.join(tmp, sub))
        ref, seqs, rows, wt = build_inputs(name, c, tmp)
        ckpt = os.path.join(tmp, "poet.ckpt")
        synth.write_poet_checkpoint(ckpt, c["arch"], seed=c["seed"])
        flags = ["--context_lengths", *map(str, c["ctx"]), "--seed", str(c.get("poet_seed", 188257)),
                 "--batch_size", str(c.get("batch_size", 8))] + (["--relative_to_wt"] if c.get("relative") else [])
        argv = ["score.py", "--checkpoint", ckpt, "--DMS_reference_file_path", os.path.join(tmp, "ref.csv"), "--DMS_data_folder",
                os.path.join(tmp, "dms"), "--DMS_index", "0", "--output_scores_folder", os.path.join(tmp, "out"), "--MSA_folder",
                os.path.join(tmp, "msa")] + flags
        rec = dict(kind="case", name=name, arch=dataclasses.asdict(c["arch"]), seed=c["seed"], ref=ref, variants=seqs, a3m=rows,
                   flags=flags, true_size=bool(c.get("true_size")))
        rec["sampler"] = sampler_record(mod, rows, wt, c["ctx"], c.get("poet_seed", 188257))
        t0 = time.time()
        old = sys.argv
        sys.argv = argv
        try:
            mod.main()
            out = pd.read_csv(os.path.join(tmp, "out", ref["DMS_filename"]))
            rec["scores"] = [None if not np.isfinite(v) else float(v) for v in out["PoET_score"]]
            rec["out_columns"] = list(out.columns)
        except Exception as e:  # noqa: BLE001
            rec["error"] = f"{type(e).__name__}: {e}"
        finally:
            sys.argv = old
        rec["cpu_seconds"] = round(time.time() - t0, 1)
    return rec


def cli_flags() -> dict:
    import argparse
    mod = R.install()
    captured = {}
    orig = argparse.ArgumentParser.parse_args

    def grab(self, *a, **k):
        captured["actions"] = [dict(dest=x.dest, option_strings=x.option_strings, default=x.default, type=getattr(x.type, "__name__", None),
                                    nargs=x.nargs, action=type(x).__name__) for x in self._actions if x.dest != "help"]
        raise SystemExit(0)
    argparse.ArgumentParser.parse_args = grab
    try:
        mod.parse_args()
    except SystemExit:
        pass
    finally:
        argparse.ArgumentParser.parse_args = orig
    return captured


def main(argv):
    if argv == ["flags"]:
        with open(FLAGS_FILE, "w") as fh:
            json.dump(cli_flags(), fh, indent=1)
        return
    names = argv or list(CASES)
    lines = {}
    if os.path.exists(GOLDEN_FILE):
        for ln in open(GOLDEN_FILE):
            r = json.loads(ln)
            lines[r["name"]] = r
    for n in names:
        r = run_case(n)
        print(n, r.get("error", ""), r["cpu_seconds"], flush=True)
        lines[n] = r
    with open(GOLDEN_FILE, "w") as fh:
        for n in CASES:
            if n in lines:
                fh.write(json.dumps(lines[n]) + "\n")


if __name__ == "__main__":
    main(sys.argv[1:])
