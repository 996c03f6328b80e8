"""PoET throughput on one GPU: seeded weights at the released shape (12 layers, 1024 wide, 16 heads), a 300-residue wild type,
``--mutants`` single mutants, and a synthetic context of 300-residue homologs filling ``--context`` tokens (24 576 by default, the
largest member of the reference's ensemble). One (context, direction) pair is timed with CUDA events: the context pass
(pg_poet_context) and the variant pass (pg_poet_loglik), each after one warm-up call. Then a separate profiled run of the same pair gives
kernel ms by category (pg_profile_*). "attention" holds the variant rows' memory attention (K17), the own-row self-attention and the
context's attention. The K17 rate is its algorithmic FLOPs, 4 * rows * layers * d * (Tm + own keys / 2), over the attention ms, quoted
against the fp16 dense peak it issues three times in the parity modes. The full 15-member ensemble is not timed here; its mutants/s is
extrapolated from the measured pair and the context lengths 6 144 / 12 288 / 24 576 and printed as such. The card and its power limit
are read in the same call.
Usage: python scripts/bench_poet.py [--precision f16x3] [--mutants 5000] [--context 24576]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from proteingym_b200 import _lib, checkpoint, synth  # noqa: E402
from proteingym_b200 import poet_engine as E  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="f16x3")
    ap.add_argument("--mutants", type=int, default=5000)
    ap.add_argument("--context", type=int, default=24576)
    ap.add_argument("--L", type=int, default=300)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_poet.py measures on a GPU"
    lib = _lib.load()
    arch = synth.POET
    st = synth.make_poet_state(arch, seed=5)
    conf = checkpoint.PoetConfig(arch.layers, arch.hidden_dim, arch.heads, 4 * arch.hidden_dim, False)
    wt = synth.random_protein(args.L, 1)
    variants = [E.append_startstop(E.encode(synth.apply_mutant(wt, m).encode())) for m in synth.sample_mutants(wt, args.mutants, 2)]
    rng = np.random.default_rng(3)
    ctx, total = [], 0
    while total <= args.context:  # the reference's overshoot: the last homolog crosses the budget
        ctx.append(E.append_startstop(rng.integers(0, 20, size=args.L).astype(np.uint8)))
        total += len(ctx[-1])
    Tm = total
    sc = E.PoetScorer(conf, st, args.L + 2, precision=args.precision)
    try:
        sc.set_context(ctx)
        sc.loglik(variants[:64])
        _, t_ctx = timed(lambda: sc.set_context(ctx))
        _, t_var = timed(lambda: sc.loglik(variants))
        ms = (C.c_float * 12)()
        cnt = (C.c_int32 * 12)()
        lib.pg_profile_begin()
        sc.set_context(ctx)
        sc.loglik(variants)
        torch.cuda.synchronize()
        lib.pg_profile_end(ms, cnt, 12)
    finally:
        sc.close()
    cats = {n: round(ms[i], 2) for i, n in enumerate(_lib.PROFILE_CATEGORIES) if cnt[i]}
    T = args.L + 2
    rows = len(variants) * (T - 1)
    d, layers = arch.hidden_dim, arch.layers
    k17_flop = 4.0 * rows * layers * d * (Tm + T / 2)
    pair_s = t_ctx + t_var
    # ensemble: 5 similarity filters x (6 144, 12 288, 24 576), each forward + backward; variant time scales with Tm + T / 2 keys
    # for the attention share, the rest is constant per pass
    att_share = cats.get("attention", 0.0) / 1e3 / max(t_var + t_ctx, 1e-9)
    est = 0.0
    for c in (6144, 12288, 24576):
        f = (c + T / 2) / (Tm + T / 2)
        est += 5 * 2 * (pair_s * (1 - att_share) + pair_s * att_share * f)
    print(json.dumps({
        "card": card(), "precision": args.precision, "context_tokens": Tm, "mutants": len(variants), "variant_tokens": T,
        "context_s": round(t_ctx, 4), "variants_s": round(t_var, 3),
        "mutants_per_s_one_pair": round(len(variants) / pair_s, 1),
        "mutants_per_s_ensemble_extrapolated": round(len(variants) / est, 2),
        "kernel_ms": cats,
        "attention_algorithmic_tflops": round(k17_flop / (cats.get("attention", float("nan")) / 1e3) / 1e12, 1),
        "attention_tflop": round(k17_flop / 1e12, 1),
    }))


if __name__ == "__main__":
    main()
