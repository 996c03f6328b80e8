"""ORACLE SUPPORT — TEST INFRASTRUCTURE ONLY. Build-container script (needs the reference tree: oracle/ref_shims.py REF).

Goldens for ESM2 8M / 35M / 150M at their true shapes: the UNMODIFIED reference CLI (oracle/gen_golden.py ``run_case``) on seeded
synthetic checkpoints, a real wild type from reference_files/DMS_substitutions.csv per release, single and 2-site mutants, and the
reference token_probs table; plus an 8M case with L + 2 > 1024 (per-position windows).   python oracle/gen_golden_esm2_small.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pandas as pd  # noqa: E402
import torch  # noqa: E402

from oracle import ref_shims  # noqa: E402
from oracle.gen_golden import run_case  # noqa: E402
from proteingym_b200 import synth  # noqa: E402

# golden name, arch, seed, DMS_id of the wild type, checkpoint file, mutants, table positions (None: all)
CASES = [
    ("esm2_8m", synth.ESM2_8M, 81, "GFP_AEQVI_Sarkisyan_2016", "esm2_t6_8M_UR50D.pt", 60, None),
    ("esm2_35m", synth.ESM2_35M, 82, "GRB2_HUMAN_Faure_2021", "esm2_t12_35M_UR50D.pt", 60, None),
    ("esm2_150m", synth.ESM2_150M, 83, "DYR_ECOLI_Thompson_2019", "esm2_t30_150M_UR50D.pt", 60, None),
    ("esm2_8m_window", synth.ESM2_8M, 84, "CAR11_HUMAN_Meitlis_2020_gof", "esm2_t6_8M_UR50D.pt", 40,
     [1, 2, 300, 511, 512, 513, 643, 644, 645, 1000, 1154]),
]

if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count() or 1)
    dms = pd.read_csv(os.path.join(ref_shims.REF, "reference_files", "DMS_substitutions.csv"))
    for k, (name, arch, seed, dms_id, ck, n, pos) in enumerate(CASES):
        seq = dms[dms["DMS_id"] == dms_id].iloc[0]["target_seq"].upper()
        run_case(name, arch, seed, seq, synth.sample_mutants(seq, n, seed=40 + k, multi_frac=0.3, max_sites=2), ck, "ESM2",
                 table_positions=pos)
