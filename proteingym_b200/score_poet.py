"""Drop-in for ``proteingym/baselines/PoET/scripts/score.py`` (PoET log-likelihoods): same flags and defaults, same output —
``<output_scores_folder>/<DMS_filename>`` with the columns mutated_sequence, PoET_score. The variants are the DMS file's
``mutated_sequence`` (or ``mutant``) strings; the MSA is ``<MSA_folder>/<DMS_filename stem>.a3m.zst`` (plain text is read as is; a
zstd-compressed file needs the pyzstd or zstandard module). ``--batch_size`` is accepted and does not change the results: the library
splits the rows into passes itself. Additive flags: ``--precision``, ``--device``."""
from __future__ import annotations

import argparse
import os
import sys
from pathlib import Path

import pandas as pd

if __package__ in (None, ""):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# --precision auto: the mode that meets the 1e-3 score bar on the PoET goldens (DESIGN.md §2)
AUTO_PRECISION = "f16x3"


def create_parser():
    p = argparse.ArgumentParser(description="PoET scoring on H100 (proteingym/baselines/PoET/scripts/score.py drop-in)")
    p.add_argument("--checkpoint", type=str, default="proteingym/baselines/PoET/scripts/data/poet.ckpt")
    p.add_argument("--DMS_reference_file_path", type=str, default="reference_files/DMS_substitutions.csv")
    p.add_argument("--DMS_data_folder", type=str, default="data/DMS_ProteinGym_substitutions")
    p.add_argument("--DMS_index", type=int, default=1)
    p.add_argument("--output_scores_folder", type=str, default="data/zero_shot_substitutions_scores/PoET")
    p.add_argument("--MSA_folder", type=str, default="proteingym/baselines/PoET/scripts/data/msas/DMS_substitutions")
    p.add_argument("--context_lengths", type=int, nargs="+", default=[6144, 12288, 24576])
    p.add_argument("--relative_to_wt", action="store_true")
    p.add_argument("--batch_size", type=int, default=8)
    p.add_argument("--seed", type=int, default=188257)
    # additive
    p.add_argument("--precision", default="auto", choices=["auto", "f16x3", "f16f8", "f16"], help="tensor-core operand scheme")
    p.add_argument("--device", type=int, default=0, help="CUDA device ordinal")
    return p


def main(args) -> pd.DataFrame:
    from proteingym_b200 import checkpoint
    from proteingym_b200 import poet_engine as E

    conf, state = checkpoint.load_poet_checkpoint(args.checkpoint)
    ref = pd.read_csv(args.DMS_reference_file_path).iloc[args.DMS_index]
    msa_start, msa_end = int(ref["MSA_start"]), int(ref["MSA_end"])
    wt_sequence = ref["target_seq"][msa_start - 1:msa_end]
    filename = ref["DMS_filename"]
    df = pd.read_csv(Path(args.DMS_data_folder) / filename)
    if "mutated_sequence" in df.columns:
        variant_sequences = df["mutated_sequence"].values
    elif "mutant" in df.columns:
        variant_sequences = df["mutant"].values
    else:
        raise ValueError("did not find sequence column in DMS file")
    variants = [E.append_startstop(E.encode(v.encode())) for v in variant_sequences]
    if args.relative_to_wt:
        variants.append(E.append_startstop(E.encode(wt_sequence.encode())))
    msa_seqs = E.parse_a3m(E.read_maybe_zstd(str((Path(args.MSA_folder) / filename).with_suffix(".a3m.zst"))))
    if msa_seqs[0].decode() != wt_sequence:
        raise AssertionError("the first MSA sequence is not the wild type (target_seq[MSA_start - 1:MSA_end])")
    msa = E.weight_matrix(msa_seqs)
    if (msa != E.GAP).sum(axis=1).min() == 0:  # the reference's sampler fails on an all-gap row before any variant is read
        E.neighbor_counts(msa, args.device)
    if any((v == E.GAP).any() for v in variants):  # the reference asserts this in its first decoding batch
        raise AssertionError("a variant contains a gap ('-')")
    longest = max(max(len(v) for v in variants), max(len(E.context_sequence(s)) + 2 for s in msa_seqs))
    precision = AUTO_PRECISION if args.precision == "auto" else args.precision
    scorer = E.PoetScorer(conf, state, longest, precision=precision, device=args.device)
    try:
        neighbors = E.neighbor_counts(msa, args.device)
        logps = E.score_members(scorer, msa_seqs, msa, neighbors, variants, args.context_lengths, args.seed)
    finally:
        scorer.close()
    if args.relative_to_wt:
        logps = logps[:-1] - logps[-1]
    out = pd.DataFrame(data={"mutated_sequence": variant_sequences, "PoET_score": logps})
    os.makedirs(args.output_scores_folder, exist_ok=True)
    out.to_csv(Path(args.output_scores_folder) / filename, index=False)
    return out


if __name__ == "__main__":
    main(create_parser().parse_args())
