"""Drop-in for ``proteingym/baselines/evoscale/compute_fitness.py`` with ``--model_type esmc_300M | esmc_600M`` (ESM C masked
marginals): same flags (:743-788), same outputs — ``<output_dir>/<DMS_id>.csv`` = the assay's columns + ``{model_type}_score``
(NaN for mutants the reference skips), and the per-assay Spearman appended to ``correlation_summary_{model_type}.csv`` (:612-740). An
exception while scoring one assay gives it a NaN correlation and no CSV, as in the reference. Additive flags: --precision, --device.
``esm3_open`` (structure and function tracks) is not implemented. Weights come from --model_path or the local Hugging Face cache; nothing
is downloaded."""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np
import pandas as pd

if __package__ in (None, ""):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def create_parser():
    p = argparse.ArgumentParser(description="ESM C masked-marginal DMS scoring on H100 (evoscale compute_fitness.py drop-in)")
    p.add_argument("--model_type", choices=["esmc_300M", "esmc_600M", "esm3_open"], default="esmc_300M", help="model to score with")
    p.add_argument("--model_path", type=str, default=None, help=".pth weights or a snapshot directory (default: local HF cache)")
    p.add_argument("--reference_csv", required=True, help="CSV with DMS_id and target_seq columns")
    p.add_argument("--dms_dir", required=True, help="directory holding <DMS_id>.csv")
    p.add_argument("--pdb_dir", required=False, default=None, help="(esm3_open with structure only)")
    p.add_argument("--output_dir", required=True, help="directory for <DMS_id>.csv and the correlation summary")
    p.add_argument("--use_structure", action="store_true", default=False, help="(esm3_open only)")
    p.add_argument("--DMS_index", required=False, default=-1, help="row of the reference CSV to score; -1 = all")
    # additive
    p.add_argument("--precision", default="auto", choices=["auto", "f16f8", "f16x3", "f16"], help="tensor-core operand scheme")
    p.add_argument("--device", type=int, default=0, help="CUDA device ordinal")
    return p


def _select(ref: pd.DataFrame, dms_index) -> pd.DataFrame:
    """compute_fitness.py:648-658: one row when the index is valid, otherwise (with a warning) every row."""
    if dms_index == -1:
        return ref
    try:
        i = int(dms_index)
    except ValueError:
        print(f"Warning: Invalid DMS_index '{dms_index}', processing all assays")
        return ref
    if 0 <= i < len(ref):
        return ref.iloc[[i]]
    print(f"Warning: DMS_index {i} out of range (0-{len(ref) - 1}), processing all assays")
    return ref


def main(args) -> dict:
    from scipy.stats import spearmanr

    if args.model_type == "esm3_open":
        raise NotImplementedError("esm3_open (structure and function tracks, geometric attention) is not implemented on this scorer")
    os.makedirs(args.output_dir, exist_ok=True)
    ref = pd.read_csv(args.reference_csv)
    if "DMS_id" not in ref.columns:
        raise ValueError("Input CSV must contain a 'DMS_id' column")
    if "target_seq" not in ref.columns:
        raise ValueError("Input CSV must contain a 'target_seq' column with protein sequences")
    if args.use_structure and "pdb_file" not in ref.columns:
        raise ValueError("Input CSV must contain a 'pdb_file' column if we use structures for scoring")
    score_col = f"{args.model_type}_score"
    scorer = {}

    def get_scorer(mutants):
        from proteingym_b200 import checkpoint
        from proteingym_b200.esm_engine import EsmScorer, choose_precision
        if "conf" not in scorer:
            scorer["conf"], scorer["state"], _ = checkpoint.load_esmc_checkpoint(args.model_type, args.model_path)
        prec = choose_precision(scorer["conf"], list(mutants)) if args.precision == "auto" else args.precision
        if scorer.get("prec") != prec:
            if "sc" in scorer:
                scorer.pop("sc").close()
            scorer["sc"] = EsmScorer(scorer["conf"], scorer["state"], precision=prec, device=args.device)
            scorer["prec"] = prec
        return scorer["sc"]

    results = {}
    for _, row in _select(ref, args.DMS_index).iterrows():
        assay, seq = row["DMS_id"], row["target_seq"]
        in_csv = os.path.join(args.dms_dir, f"{assay}.csv")
        if not os.path.exists(in_csv):
            print(f"Error: Input CSV file {in_csv} not found, skipping")
            continue
        try:
            df = pd.read_csv(in_csv)
            mutants = df["mutant"].tolist()
            if len(seq) == 0:
                raise ValueError("Empty sequence provided")
            df[score_col] = get_scorer(mutants).score_assay(seq, mutants).astype(np.float64)
            valid = df.dropna(subset=[score_col, "DMS_score"])
            corr = spearmanr(valid["DMS_score"], valid[score_col])[0] if len(valid) > 0 else np.nan
            df.to_csv(os.path.join(args.output_dir, f"{assay}.csv"), index=False)
            results[assay] = corr
        except Exception as e:  # compute_fitness.py:724-726
            print(f"Error processing {assay}: {e}")
            results[assay] = np.nan
    if "sc" in scorer:
        scorer["sc"].close()
    summary = pd.DataFrame({"assay": list(results.keys()), "correlation": list(results.values())})
    path = os.path.join(args.output_dir, f"correlation_summary_{args.model_type}.csv")
    if os.path.exists(path):
        summary.to_csv(path, mode="a", header=False, index=False)
    else:
        summary.to_csv(path, index=False)
    return results


if __name__ == "__main__":
    main(create_parser().parse_args())
