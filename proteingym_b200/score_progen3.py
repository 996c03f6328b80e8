"""Drop-in for ``proteingym/baselines/progen3/progen3/tools/score.py`` (ProGen3 log-likelihoods of the sequences of a FASTA file): same
flags (:12-28), same output — a CSV indexed by ``sequence_id`` (the FASTA record ids, sorted) with the columns ``log_likelihood`` and
``perplexity`` written from float32 values as ``ProGen3Scorer.run`` writes them (scorer.py:169-182).

``--model-name`` is a local model directory (config.json + *.safetensors or pytorch_model.bin, eager or megablocks layout): nothing is
downloaded. ``--max-batch-tokens`` and ``--seed`` are accepted; neither changes a score (batches are right-padded and causal, and scoring
draws no random numbers). ``--fsdp`` is accepted and has no effect on scores: the model runs on one GPU. The reference loads the weights
in bf16; this scorer runs them at ``--precision`` (the tensor-core operand scheme, default f16f8) on fp32 weights, and its parity bar is
the reference run in fp32. Additive flags: ``--precision``, ``--device``."""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np
import pandas as pd

if __package__ in (None, ""):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def create_parser():
    p = argparse.ArgumentParser(description="ProGen3 scoring on H100 (progen3/tools/score.py drop-in)")
    p.add_argument("--model-name", dest="model_name", type=str, required=True, help="ProGen3 model directory")
    p.add_argument("--fasta-path", dest="fasta_path", type=str, required=True, help="FASTA file of the sequences to score")
    p.add_argument("--output-path", dest="output_path", type=str, required=True, help="CSV to write")
    p.add_argument("--max-batch-tokens", dest="max_batch_tokens", type=int, default=65536,
                   help="accepted for compatibility; batching does not change scores")
    p.add_argument("--fsdp", dest="fsdp", action="store_true", help="accepted for compatibility; no effect on scores (one GPU)")
    p.add_argument("--seed", dest="seed", type=int, default=42, help="accepted for compatibility; scoring draws no random numbers")
    # additive
    p.add_argument("--precision", default="f16f8", choices=["f16f8", "f16x3", "f16"], help="tensor-core operand scheme")
    p.add_argument("--device", type=int, default=0, help="CUDA device ordinal")
    return p


def main(args) -> pd.DataFrame:
    from proteingym_b200 import checkpoint
    from proteingym_b200.progen3_engine import MAX_POSITIONS, Progen3Scorer, read_fasta

    seqs = read_fasta(args.fasta_path)
    ids = sorted(seqs)
    conf, state = checkpoint.load_progen3_checkpoint(args.model_name)
    longest = max((len(seqs[i]) for i in ids), default=0) + 4
    sc = Progen3Scorer(conf, state, precision=args.precision, device=args.device, max_positions=max(MAX_POSITIONS, longest))
    try:
        ll, ppl = sc.score([seqs[i] for i in ids])
    finally:
        sc.close()
    df = pd.DataFrame({"log_likelihood": ll.astype(np.float32), "perplexity": ppl.astype(np.float32)}, index=ids)
    df.index.name = "sequence_id"
    df.to_csv(args.output_path)
    return df


if __name__ == "__main__":
    main(create_parser().parse_args())
