"""Drop-in for ``proteingym/baselines/progen2/compute_fitness.py`` (ProGen2 small / medium / base / large log-likelihoods): same flags
(:117-124), same output — ``<output_scores_folder>/<DMS_id>.csv`` with the columns mutant, Progen2_score, DMS_score (:165-167). In
substitution mode a DMS file without a ``mutated_sequence`` column gets one from the mutant strings, wrapped in the terminals as
``"1" + sequence + "2"`` (get_mutated_sequence, :88-103, same assertions); an existing column, and ``--indel_mode``, are scored as given.
The chunk length is the checkpoint's ``n_positions`` (:163).

``--fp16`` is accepted for compatibility; the scoring precision is ``--precision`` (the tensor-core operand scheme, default f16f8,
whatever the checkpoint's stored dtype: weights are upcast to fp32 at load). ``--test`` checks the released weights' log-likelihood of
built-in sequences against constants of the reference script, which are not reproduced here: it raises NotImplementedError. Additive
flags: ``--precision``, ``--device``. Nothing is downloaded."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import pandas as pd

if __package__ in (None, ""):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def create_parser():
    p = argparse.ArgumentParser(description="ProGen2 scoring on H100 (proteingym/baselines/progen2/compute_fitness.py drop-in)")
    p.add_argument("--Progen2_model_name_or_path", default="/n/groups/marks/projects/marks_lab_and_oatml/protein_transformer/baseline_models/progen2/progen2-small",
                   type=str, help="ProGen2 model directory (config.json + pytorch_model.bin or *.safetensors)")
    p.add_argument("--DMS_reference_file_path", default="/home/pn73/Tranception/proteingym/ProteinGym_reference_file_substitutions.csv", type=str,
                   help="reference file (DMS_id, DMS_filename, target_seq)")
    p.add_argument("--DMS_data_folder", default="/n/groups/marks/projects/marks_lab_and_oatml/protein_transformer/Tranception_open_source/DMS_files/ProteinGym_substitutions",
                   type=str, help="folder of the DMS files")
    p.add_argument("--DMS_index", type=int, help="row of the reference file to score")
    p.add_argument("--output_scores_folder", default=None, type=str, help="folder to write <DMS_id>.csv to")
    p.add_argument("--indel_mode", action="store_true", help="score mutated_sequence as given (insertions and deletions)")
    p.add_argument("--fp16", action="store_true", help="accepted for compatibility; the scoring precision is --precision")
    p.add_argument("--test", action="store_true", help="the reference's released-weights check (not implemented)")
    # additive
    p.add_argument("--precision", default="f16f8", choices=["f16f8", "f16x3", "f16"], help="tensor-core operand scheme")
    p.add_argument("--device", type=int, default=0, help="CUDA device ordinal")
    return p


def main(args) -> pd.DataFrame:
    from proteingym_b200 import checkpoint
    from proteingym_b200.progen2_engine import Progen2Scorer
    from proteingym_b200.tranception_engine import apply_substitutions

    if args.test:
        raise NotImplementedError("--test compares the released checkpoints with log-likelihood constants of the reference script, "
                                  "which this drop-in does not reproduce")
    conf, state = checkpoint.load_progen2_checkpoint(args.Progen2_model_name_or_path)
    with open(os.path.join(args.Progen2_model_name_or_path, "config.json")) as fh:
        print("Maximum context length: {}".format(json.load(fh)["n_positions"]))
    ref = pd.read_csv(args.DMS_reference_file_path)
    DMS_id = ref["DMS_id"][args.DMS_index]
    print("Computing scores for: {} with Progen2: {}".format(DMS_id, args.Progen2_model_name_or_path))
    DMS_file_name = ref["DMS_filename"][ref["DMS_id"] == DMS_id].values[0]
    target_seq = ref["target_seq"][ref["DMS_id"] == DMS_id].values[0].upper()
    DMS_data = pd.read_csv(args.DMS_data_folder + os.sep + DMS_file_name, low_memory=False)
    wt = target_seq
    if not args.indel_mode and "mutated_sequence" not in DMS_data.columns:
        DMS_data["mutated_sequence"] = DMS_data["mutant"].apply(lambda x: "1" + apply_substitutions(target_seq, x) + "2")
        wt = "1" + target_seq + "2"
    sc = Progen2Scorer(conf, state, precision=args.precision, device=args.device)
    try:
        DMS_data["Progen2_score"] = sc.score(list(np.array(DMS_data["mutated_sequence"])), wt=wt)
    finally:
        sc.close()
    out = DMS_data[["mutant", "Progen2_score", "DMS_score"]]
    out.to_csv(args.output_scores_folder + os.sep + DMS_id + ".csv", index=False)
    return out


if __name__ == "__main__":
    main(create_parser().parse_args())
