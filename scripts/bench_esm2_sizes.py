"""ESM2 throughput by release (8M / 35M / 150M in 64-wide head slots, 650M for comparison): masked-marginal scoring of an L = 512
protein with 5000 single mutants per step, seeded weights at the true shapes. One JSON line per release and precision: mutants/s over
`--steps` device-resident steps (CUDA events), per-category kernel ms of one profiled step (pg_profile_*), and the linear / attention
FLOPs of a step counted from shapes, padded (as run, DESIGN.md §3) and unpadded (as the model defines them), with the card and its
power limit.   python scripts/bench_esm2_sizes.py [--steps 5] [--warmup 2] [--releases 8m,35m,150m,650m] [--precisions f16x3,f16f8]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from proteingym_b200 import _lib, checkpoint, synth  # noqa: E402
from proteingym_b200.esm_engine import EsmScorer  # noqa: E402

RELEASES = {"8m": synth.ESM2_8M, "35m": synth.ESM2_35M, "150m": synth.ESM2_150M, "650m": synth.ESM2_650M}


def flops(arch, T, P, padded):
    """(linear, attention) FLOPs of P masked copies of a T-token window; the pruned last layer runs q/k/v on all rows, the rest on P."""
    d, f, n = arch.embed_dim, arch.ffn_dim, arch.layers
    da, dk = (arch.heads * 64, (d + 63) // 64 * 64) if padded else (d, d)
    qkv, rest = 3 * da * dk, da * d + dk * f + f * d
    return 2 * ((n - 1) * P * T * (qkv + rest) + P * T * qkv + P * rest), 4 * da * ((n - 1) * P * T * T + P * T)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--releases", default="8m,35m,150m,650m")
    ap.add_argument("--precisions", default="f16x3,f16f8")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_esm2_sizes: no CUDA device")
    lib = _lib.load()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                          text=True).stdout.strip()
    seq = synth.random_protein(512, 0)
    muts = synth.sample_mutants(seq, 5000, 1000)
    for rel in a.releases.split(","):
        arch = RELEASES[rel]
        state = checkpoint.normalise_synth_state(arch, synth.make_esm_state(arch, seed=0, device="cuda"))
        for prec in a.precisions.split(","):
            sc = EsmScorer(checkpoint.config_from_synth(arch), state, precision=prec)
            host, sizes = sc.prepare_assay(seq, muts)
            dev = host.to(sc.device)
            for _ in range(a.warmup):
                sc.run_assay(host, sizes, dev=dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                sc.run_assay(host, sizes, dev=dev)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / a.steps
            lib.pg_profile_begin()
            sc.run_assay(host, sizes, dev=dev)
            torch.cuda.synchronize()
            n = len(_lib.PROFILE_CATEGORIES)
            cat_ms, cat_n = (C.c_float * n)(), (C.c_int32 * n)()
            lib.pg_profile_end(cat_ms, cat_n, n)
            sc.close()
            cats = {c: round(float(cat_ms[i]), 3) for i, c in enumerate(_lib.PROFILE_CATEGORIES) if cat_n[i]}
            fp, fu = flops(arch, sizes["T"], sizes["P"], True), flops(arch, sizes["T"], sizes["P"], False)
            print(json.dumps({"release": f"esm2_{rel}", "precision": prec, "ms_per_step": round(ms, 3),
                              "mutants_per_s": round(len(muts) / (ms / 1e3), 1),
                              "kernel_ms": {"gemm": round(sum(v for c, v in cats.items() if c.startswith("gemm")), 3),
                                            "attention": cats.get("attention"), "layernorm": cats.get("layernorm"), "all": cats},
                              "flops_linear": {"padded": fp[0], "unpadded": fu[0]}, "flops_attention": {"padded": fp[1], "unpadded": fu[1]},
                              "card": card}), flush=True)
        del state
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
