"""ProGen2 small / medium / large throughput on one GPU: seeded weights at true size, a 512-residue wild type and 5 000 single mutants,
scored as calc_fitness scores them (both directions, one chunk, the raw sequences of a DMS file's mutated_sequence column) with
wild-type prefix reuse on and off. One JSON line per model and precision: mutants/s (CUDA events around Progen2Scorer.score,
tokenisation and planning included), token rows run with and without reuse, kernel ms by category (pg_profile_*, from a separate
profiled run without prefix reuse, so that every row is a full 512-token row), algorithmic GEMM TFLOP/s (2 * rows * (3d*d + d*d +
2*d*f) over the GEMM ms) and attention TFLOP/s counted at the model's head_dim (4 * heads * head_dim * T(T+1)/2 per row and layer; the
zero columns of a 128-wide head slot are not work), and the card with its power limit, read in the same call.
Usage: python scripts/bench_progen2.py [--models small medium large] [--precisions f16f8] [--mutants 5000] [--L 512]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from proteingym_b200 import _lib, checkpoint, synth  # noqa: E402
from proteingym_b200.progen2_engine import Progen2Scorer  # noqa: E402

ARCHS = {"small": synth.PROGEN2_SMALL, "medium": synth.PROGEN2_MEDIUM, "large": synth.PROGEN2_LARGE}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def timed(sc, prots, wt):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    out = sc.score(prots, wt=wt)
    end.record()
    torch.cuda.synchronize()
    return out, start.elapsed_time(end) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=list(ARCHS))
    ap.add_argument("--precisions", nargs="+", default=["f16f8"])
    ap.add_argument("--mutants", type=int, default=5000)
    ap.add_argument("--L", type=int, default=512)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_progen2.py measures on a GPU"
    lib = _lib.load()
    gpu = card()
    wt = synth.random_protein(args.L, 1)
    prots = [synth.apply_mutant(wt, m) for m in synth.sample_mutants(wt, args.mutants, 2)]
    for name in args.models:
        arch = ARCHS[name]
        st = synth.make_progen2_state(arch, seed=3, buffers=False)
        ws = {k[len("transformer."):] if k.startswith("transformer.") else k: v for k, v in st.items()}
        del st
        conf = checkpoint.Progen2Config(arch.layers, arch.embed_dim, arch.heads, arch.ffn_dim, arch.vocab, arch.rotary_dim, arch.n_positions)
        for prec in args.precisions:
            sc = Progen2Scorer(conf, ws, precision=prec)
            res = {}
            for reuse in (True, False):
                sc.prefix_reuse = reuse
                timed(sc, prots[:64], wt)  # warm-up of every shape class
                sc.reuse_rows = [0, 0]
                out, sec = timed(sc, prots, wt)
                res[reuse] = (out, sec, list(sc.reuse_rows))
            ms = (C.c_float * 12)()
            cnt = (C.c_int32 * 12)()
            lib.pg_profile_begin()
            sc.score(prots, wt=wt)  # prefix reuse off: full rows
            torch.cuda.synchronize()
            lib.pg_profile_end(ms, cnt, 12)
            cats = {c: round(ms[i], 2) for i, c in enumerate(_lib.PROFILE_CATEGORIES) if ms[i] > 0}
            gemm_ms = sum(cats.get(c, 0.0) for c in ("gemm_qkv", "gemm_out", "gemm_fc1", "gemm_fc2"))
            d, f, T = arch.embed_dim, arch.ffn_dim, args.L
            rows_run = res[False][2][1]
            flops = 2.0 * rows_run * arch.layers * (4 * d * d + 2 * d * f)
            attn_flops = 4.0 * arch.heads * arch.head_dim * (T * (T + 1) / 2) * (rows_run / T) * arch.layers
            diff = float(np.max(np.abs(res[True][0] - res[False][0])))
            print(json.dumps(dict(model=f"progen2-{name}", head_dim=arch.head_dim, precision=prec, L=args.L, mutants=len(prots),
                                  mutants_per_s_reuse=round(len(prots) / res[True][1], 1), mutants_per_s_plain=round(len(prots) / res[False][1], 1),
                                  token_rows_plain=res[True][2][0], token_rows_run_reuse=res[True][2][1], token_rows_run_plain=rows_run,
                                  max_score_diff_reuse_vs_plain=diff, kernel_ms=cats, gemm_tflops=round(flops / (gemm_ms * 1e-3) / 1e12, 1),
                                  attention_tflops=round(attn_flops / (cats.get("attention", float("nan")) * 1e-3) / 1e12, 1),
                                  gpu=gpu)), flush=True)
            sc.close()
        del ws
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
