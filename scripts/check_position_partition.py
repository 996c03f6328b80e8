"""torchrun --nproc-per-node N scripts/check_position_partition.py: one assay scored with its masked positions split over N GPUs
(EsmScorer.score_assay(shard=...)) must equal, bit for bit, the single-GPU scores rank 0 computes alone. Prints one line."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from proteingym_b200 import sharding, synth  # noqa: E402
from proteingym_b200.checkpoint import config_from_synth, normalise_synth_state  # noqa: E402
from proteingym_b200.esm_engine import EsmScorer  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    which = sys.argv[1] if len(sys.argv) > 1 else ""
    big = which == "650m"
    arch = {"650m": synth.ESM1V_650M, "esm2_8m": synth.ESM2_8M}.get(which, synth.EsmArch("esm1v", 3, 256, 4, 1024))
    conf = config_from_synth(arch)
    state = sharding.broadcast_state(normalise_synth_state(arch, synth.make_esm_state(arch, seed=0)) if rank == 0 else None, src=0,
                                     device=torch.device("cuda", local))
    sc = EsmScorer(conf, state, device=local)
    seq = synth.random_protein(512 if big else 203, 1)
    muts = synth.sample_mutants(seq, 5000 if big else 700, 2, multi_frac=0.2)
    torch.cuda.synchronize()
    dist.barrier()
    t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    split = sc.score_assay(seq, muts, shard=(rank, world))
    t1.record(); torch.cuda.synchronize()
    ms_split = t0.elapsed_time(t1)
    ok = True
    if rank == 0:
        t0.record()
        alone = sc.score_assay(seq, muts)
        t1.record(); torch.cuda.synchronize()
        ok = bool(np.array_equal(split, alone))
        print(f"position-partition world={world} mutants={len(muts)} L={len(seq)} bit_identical={ok} ms_split={ms_split:.1f} ms_alone={t0.elapsed_time(t1):.1f}", flush=True)
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    sc.close()
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()
