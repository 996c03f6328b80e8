"""ORACLE SUPPORT — regenerates the ProGen3 goldens by running the UNMODIFIED ProGen3ForCausalLM + ProGen3Scorer.evaluate (reference root
proteingym/baselines/progen3/progen3) on the CPU in fp32, through oracle/ref_shims_progen3.py, on seeded synthetic weights
(synth.make_progen3_state, eager layout). Writes tests/golden/progen3_goldens.jsonl: per case the seed, the arch, the FASTA records
(id -> sequence), CPU seconds, and either the CSV text ProGen3Scorer.run would write for them (DataFrame(scores, index=sorted ids),
index "sequence_id") or the exception the reference raised; and tests/golden/progen3_cli_flags.json, the options of tools/score.py.
Usage: python oracle/gen_golden_progen3.py"""
from __future__ import annotations

import dataclasses
import io
import json
import os
import sys
import time

import numpy as np
import pandas as pd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims_progen3 as R  # noqa: E402
from proteingym_b200 import synth  # noqa: E402

GOLDEN_FILE = os.path.join(ROOT, "tests", "golden", "progen3_goldens.jsonl")
FLAGS_FILE = os.path.join(ROOT, "tests", "golden", "progen3_cli_flags.json")
A = synth.Progen3Arch


def _records(seed: int, lengths, extra=()):
    rng = np.random.default_rng(seed)
    recs = {f"seq_{i:03d}": "".join(rng.choice(list(synth.AA20), n)) for i, n in enumerate(lengths)}
    recs.update(dict(extra))
    return recs


CASES = {
    # hd 64, GQA 4:2, 8 experts top-2, SiLU experts; odd characters the tokenizer drops or keeps (B J O U X Z are vocabulary letters)
    "tiny": dict(arch=A(2, 256, 4, 2, 512), seed=11, lengths=[1, 2, 7, 33, 64, 65, 130],
                 extra={"odd_letters": "ACBJOUXZDE", "dropped": "acdefGHIK*-"}),
    "gated_hd128": dict(arch=A(2, 512, 4, 2, 256, gated_mlp=True), seed=12, lengths=[5, 62, 63, 126, 200]),
    "one_expert": dict(arch=A(2, 256, 4, 4, 256, n_experts=1, top_k=1), seed=13, lengths=[3, 60, 125]),
    "top4_of_6_gated": dict(arch=A(2, 256, 4, 1, 256, n_experts=6, top_k=4, gated_mlp=True), seed=14, lengths=[9, 100]),
    # n_experts == top_k: the reference's dense branch (moe.py:99-104) stacks 3-D expert outputs into a 4-D tensor and einsum fails
    "dense_all_experts": dict(arch=A(2, 256, 4, 2, 256, n_experts=4, top_k=4), seed=15, lengths=[10]),
    "deep_24x1024": dict(arch=A(24, 1024, 16, 4, 512, n_experts=4, top_k=2), seed=16, lengths=[20, 140]),
}


def run_case(name: str) -> dict:
    c = CASES[name]
    arch = c["arch"]
    recs = _records(c["seed"], c["lengths"], c.get("extra", {}).items())
    st = synth.make_progen3_state(arch, c["seed"])
    out = dict(kind="case", name=name, seed=c["seed"], arch=dataclasses.asdict(arch), records=recs)
    t = time.time()
    try:
        sc = R.scorer(R.load_model(arch.config(), st))
        ids = sorted(recs)
        scores = sc.evaluate([recs[i] for i in ids])
        df = pd.DataFrame(scores, index=ids)
        df.index.name = "sequence_id"
        buf = io.StringIO()
        df.to_csv(buf)
        out["csv"] = buf.getvalue()
        out["log_likelihood"] = [float(v) for v in scores["log_likelihood"]]
    except Exception as e:  # the reference's own failure is the golden
        out["error"] = f"{type(e).__name__}: {e}"
    out["cpu_seconds"] = round(time.time() - t, 2)
    return out


def cli_flags() -> dict:
    R.install()
    from progen3.tools import score as S
    return {"options": [dict(name=p.name, opts=list(p.opts), default=p.default, is_flag=bool(getattr(p, "is_flag", False)),
                             required=bool(p.required), type=p.type.name) for p in S.score.params]}


def main():
    with open(GOLDEN_FILE, "w") as fh:
        for name in CASES:
            r = run_case(name)
            print(name, r.get("error", ""), r["cpu_seconds"], flush=True)
            fh.write(json.dumps(r) + "\n")
    with open(FLAGS_FILE, "w") as fh:
        json.dump(cli_flags(), fh, indent=1)


if __name__ == "__main__":
    main()
