"""ProtGPT2 throughput on one GPU: seeded weights at true size (36 layers, 1280 wide, 20 heads, 50 257 tokens), the fixture byte-level
BPE tokenizer (tests/golden/protgpt2_tokenizer), a 512-residue wild type and 5 000 single mutants, scored as calc_fitness scores them
(both directions, one chunk) with wild-type prefix reuse on and off. One JSON line per precision: mutants/s (CUDA events around
Protgpt2Scorer.score, tokenisation and planning included), the tokenisation seconds on the host, token rows run with and without reuse,
kernel ms by category (pg_profile_*, from a separate profiled run without prefix reuse; "head" is the fused LM head K16 with its ln_f
and combine kernels), algorithmic GEMM TFLOP/s of the blocks (2 * rows * (4d^2 + 2df) over the GEMM ms) and of the head
(2 * rows * d * 50 257 over the head ms), and the card with its power limit, read in the same call.
Usage: python scripts/bench_protgpt2.py [--precisions f16f8] [--mutants 5000] [--L 512]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from proteingym_b200 import _lib, checkpoint, synth  # noqa: E402
from proteingym_b200.protgpt2_engine import Protgpt2Scorer, Protgpt2Tokenizer  # noqa: E402
from proteingym_b200.decoder import plan  # noqa: E402

TOK_DIR = os.path.join(ROOT, "tests", "golden", "protgpt2_tokenizer")


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
    ap.add_argument("--precisions", nargs="+", default=["f16f8"])
    ap.add_argument("--mutants", type=int, default=5000)
    ap.add_argument("--L", type=int, default=512)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_protgpt2.py measures on a GPU"
    lib = _lib.load()
    gpu = card()
    tok = Protgpt2Tokenizer(TOK_DIR)
    wt = synth.random_protein(args.L, 1)
    prots = [synth.apply_mutant(wt, m) for m in synth.sample_mutants(wt, args.mutants, 2)]
    rows, _, _ = plan(prots, wt)
    t0 = time.perf_counter()
    toks = [tok.encode(s) for s in rows]
    tok_s = time.perf_counter() - t0
    arch = synth.PROTGPT2
    st = synth.make_protgpt2_state(arch, seed=3)
    ws = {k[len("transformer."):] if k.startswith("transformer.") else k: v for k, v in st.items() if k != "lm_head.weight"}
    del st
    conf = checkpoint.Protgpt2Config(arch.layers, arch.embed_dim, arch.heads, arch.ffn_dim, arch.vocab, arch.n_positions)
    for prec in args.precisions:
        sc = Protgpt2Scorer(conf, ws, tok, precision=prec)
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
        d, f = arch.embed_dim, arch.ffn_dim
        rows_run = res[False][2][1]
        flops = 2.0 * rows_run * arch.layers * (4 * d * d + 2 * d * f)
        head_flops = 2.0 * rows_run * d * arch.vocab
        diff = float(np.max(np.abs(res[True][0] - res[False][0])))
        print(json.dumps(dict(model="protgpt2", precision=prec, L=args.L, mutants=len(prots), mean_tokens_per_row=round(float(np.mean([len(t) for t in toks])), 1),
                              tokenise_s=round(tok_s, 3), tokenise_rows=len(rows),
                              mutants_per_s_reuse=round(len(prots) / res[True][1], 1), mutants_per_s_plain=round(len(prots) / res[False][1], 1),
                              token_rows_plain=res[True][2][0], token_rows_run_reuse=res[True][2][1], token_rows_run_plain=rows_run,
                              max_score_diff_reuse_vs_plain=diff, kernel_ms=cats, gemm_tflops=round(flops / (gemm_ms * 1e-3) / 1e12, 1),
                              head_tflops=round(head_flops / (cats.get("head", float("nan")) * 1e-3) / 1e12, 1), gpu=gpu)), flush=True)
        sc.close()


if __name__ == "__main__":
    main()
