"""ESM C throughput (300M and 600M): masked-marginal scoring of an L = 512 protein with 5000 single mutants per step, seeded weights at
the true shapes. One JSON line per release and precision: device-resident mutants/s over `--steps` steps (CUDA events), per-category
kernel ms of one profiled step (pg_profile_*; the q/k LayerNorm + rotary kernel counts as layernorm), and the algorithmic GEMM TFLOP/s
from shapes, layers * 2 * T * (4 d^2 + 3 d f) per masked copy, with the card and its power limit.
   python scripts/bench_esmc.py [--steps 5] [--warmup 2] [--releases 300m,600m] [--precisions f16f8,f16x3]"""
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

RELEASES = {"300m": synth.ESMC_300M, "600m": synth.ESMC_600M}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--releases", default="300m,600m")
    ap.add_argument("--precisions", default="f16f8,f16x3")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_esmc: no CUDA device")
    lib = _lib.load()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                          text=True).stdout.strip()
    seq = synth.random_protein(512, 0)
    muts = synth.sample_mutants(seq, 5000, 1000)
    for rel in a.releases.split(","):
        arch = RELEASES[rel]
        state = synth.make_esmc_state(arch, seed=0)
        conf = checkpoint.esmc_config_from_state(state)
        for prec in a.precisions.split(","):
            sc = EsmScorer(conf, state, precision=prec)
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
            d, f, T, P = arch.embed_dim, arch.ffn_dim, sizes["T"], sizes["P"]
            gemm_flops = arch.layers * 2 * T * (4 * d * d + 3 * d * f) * P
            print(json.dumps({"release": f"esmc_{rel}", "precision": prec, "ms_per_step": round(ms, 3),
                              "mutants_per_s": round(len(muts) / (ms / 1e3), 1), "masked_copies": P, "T": T,
                              "gemm_tflops_algorithmic": round(gemm_flops / (ms / 1e3) / 1e12, 1),
                              "kernel_ms": cats, "card": card}), flush=True)
        del state


if __name__ == "__main__":
    main()
