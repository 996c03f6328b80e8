"""Drop-in for ``proteingym/baselines/protgpt2/compute_fitness.py`` (ProtGPT2 log-likelihoods): same flags (:63-71), same output —
``<output_scores_folder>/<DMS_id>.csv`` with the columns mutated_sequence, ProtGPT2_score, DMS_score (:93-95). Substitutions get
``mutated_sequence`` from the mutant strings (get_mutated_sequence, :45-60, same assertions) unless the column exists; ``--indel_mode``
scores the column as given. The tokenizer is read from the model directory (the reference hard-codes a cluster path, :77). Additive
flags: ``--precision``, ``--device``. Nothing is downloaded."""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np
import pandas as pd

if __package__ in (None, ""):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def create_parser():
    p = argparse.ArgumentParser(description="ProtGPT2 scoring on H100 (proteingym/baselines/protgpt2/compute_fitness.py drop-in)")
    p.add_argument("--ProtGPT2_model_name_or_path", default="./", type=str,
                   help="ProtGPT2 model directory (config.json, pytorch_model.bin or *.safetensors, tokenizer.json or vocab.json + merges.txt)")
    p.add_argument("--DMS_reference_file_path", default="./proteingym/ProteinGym_reference_file_substitutions.csv", type=str,
                   help="reference file (DMS_id, DMS_filename, target_seq)")
    p.add_argument("--DMS_data_folder", default="./DMS_files/ProteinGym_substitutions", type=str, help="folder of the DMS files")
    p.add_argument("--DMS_index", type=int, help="row of the reference file to score")
    p.add_argument("--output_scores_folder", default=None, type=str, help="folder to write <DMS_id>.csv to")
    p.add_argument("--indel_mode", action="store_true", help="score mutated_sequence as given (insertions and deletions)")
    # additive
    p.add_argument("--precision", default="f16f8", choices=["f16f8", "f16x3", "f16"], help="tensor-core operand scheme")
    p.add_argument("--device", type=int, default=0, help="CUDA device ordinal")
    return p


def main(args) -> pd.DataFrame:
    from proteingym_b200 import checkpoint
    from proteingym_b200.protgpt2_engine import Protgpt2Scorer, Protgpt2Tokenizer
    from proteingym_b200.tranception_engine import apply_substitutions

    tokenizer = Protgpt2Tokenizer(args.ProtGPT2_model_name_or_path)
    conf, state = checkpoint.load_protgpt2_checkpoint(args.ProtGPT2_model_name_or_path)
    ref = pd.read_csv(args.DMS_reference_file_path)
    DMS_id = ref["DMS_id"][args.DMS_index]
    print("Computing scores for: {} with ProtGPT2: {}".format(DMS_id, args.ProtGPT2_model_name_or_path))
    DMS_file_name = ref["DMS_filename"][ref["DMS_id"] == DMS_id].values[0]
    target_seq = ref["target_seq"][ref["DMS_id"] == DMS_id].values[0].upper()
    DMS_data = pd.read_csv(args.DMS_data_folder + os.sep + DMS_file_name, low_memory=False)
    if not args.indel_mode and "mutated_sequence" not in DMS_data.columns:
        DMS_data["mutated_sequence"] = DMS_data["mutant"].apply(lambda x: apply_substitutions(target_seq, x))
    sc = Protgpt2Scorer(conf, state, tokenizer, precision=args.precision, device=args.device)
    try:
        DMS_data["ProtGPT2_score"] = sc.score(list(np.array(DMS_data["mutated_sequence"])), wt=target_seq)
    finally:
        sc.close()
    out = DMS_data[["mutated_sequence", "ProtGPT2_score", "DMS_score"]]
    out.to_csv(args.output_scores_folder + os.sep + DMS_id + ".csv", index=False)
    return out


if __name__ == "__main__":
    main(create_parser().parse_args())
