"""ProGen3 throughput on one GPU: seeded weights of a synthetic ProGen3 shape (the released models' shapes are not in the reference
tree), a 512-residue wild type and its single mutants, every sequence scored in both directions as ProGen3Scorer does. One JSON line
per precision and expert-segment height (pg_set_tuning "moe_pad": 128 runs the experts' grouped GEMMs single-CTA, 256 as two-CTA
clusters): mutants/s (CUDA events around Progen3Scorer.score, tokenisation included; warmed up first), kernel ms by category
(pg_profile_*, a separate profiled run: "layernorm" = RMSNorm before attention, "other" = router + combine, "regroup" = rank / scan /
permute, "gemm_fc1" / "gemm_fc2" = the experts' ragged grouped GEMMs), the algorithmic MoE GEMM TFLOP/s (2 * tokens * top_k * (d * n1 +
f * d) over the fc1 + fc2 ms, n1 = f or 2f gated; padding rows are not work), and the card with its power limit, read in the same call.
Usage: python scripts/bench_progen3.py [--precisions f16f8 f16x3 f16] [--mutants 1000] [--L 512]"""
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
from proteingym_b200.progen3_engine import Progen3Scorer  # noqa: E402

ARCH = synth.Progen3Arch(layers=12, embed_dim=1024, heads=16, kv_heads=4, ffn_dim=1024, n_experts=8, top_k=2, gated_mlp=True)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def timed(sc, prots):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    out = sc.score(prots)
    end.record()
    torch.cuda.synchronize()
    return out, start.elapsed_time(end) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precisions", nargs="+", default=["f16f8", "f16x3", "f16"])
    ap.add_argument("--pads", nargs="+", type=int, default=[128, 256])
    ap.add_argument("--mutants", type=int, default=1000)
    ap.add_argument("--L", type=int, default=512)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_progen3.py measures on a GPU"
    lib = _lib.load()
    gpu = card()
    wt = synth.random_protein(args.L, 1)
    prots = [synth.apply_mutant(wt, m) for m in synth.sample_mutants(wt, args.mutants, 2, multi_frac=0.0)]
    conf = checkpoint.progen3_config(ARCH.config())
    st = checkpoint.normalise_progen3_state(conf, synth.make_progen3_state(ARCH, 3))
    d, f, k = conf.embed_dim, conf.ffn_dim, conf.top_k
    n1 = 2 * f if conf.gated_mlp else f
    for prec in args.precisions:
        sc = Progen3Scorer(conf, st, precision=prec)
        ref = None
        for pad in args.pads:
            _lib.check(lib.pg_set_tuning(b"moe_pad", pad))
            timed(sc, prots[:64])
            (ll, _), sec = timed(sc, prots)
            ref = ll if ref is None else ref
            ms = (C.c_float * 12)()
            cnt = (C.c_int32 * 12)()
            lib.pg_profile_begin()
            sc.score(prots)
            torch.cuda.synchronize()
            lib.pg_profile_end(ms, cnt, 12)
            cats = {c: round(ms[i], 2) for i, c in enumerate(_lib.PROFILE_CATEGORIES) if ms[i] > 0}
            tokens = 2 * len(prots) * (args.L + 4)
            moe_flops = 2.0 * tokens * k * (d * n1 + f * d) * conf.layers
            moe_ms = cats.get("gemm_fc1", 0.0) + cats.get("gemm_fc2", 0.0)
            print(json.dumps(dict(arch=ARCH.__dict__, precision=prec, moe_pad=pad, L=args.L, mutants=len(prots),
                                  mutants_per_s=round(len(prots) / sec, 1), kernel_ms=cats,
                                  moe_gemm_tflops=round(moe_flops / (moe_ms * 1e-3) / 1e12, 1) if moe_ms else None,
                                  max_ll_diff_vs_first_pad=float(np.max(np.abs(ll - ref))), gpu=gpu)), flush=True)
        _lib.check(lib.pg_set_tuning(b"moe_pad", 128))
        sc.close()


if __name__ == "__main__":
    main()
