"""Worker of tests/test_gpu_dist_between_steps.py: one rank (one GPU) of a sharded run with calls between its steps
(push_pull, remove_dead_nodes, add_members, join, leave). It replays the phase list of case.npz: phase k steps
before[k] rounds, makes calls[k] with its arguments, then steps each nonzero chunk of after[k] and takes the digest
after each. The call's totals and the digests are summed over the ranks; rank 0 writes them and the gathered state
arrays."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch.distributed as dist  # noqa: E402

from swim_b200 import _abi as A  # noqa: E402
from swim_b200 import dist as sdist  # noqa: E402
from swim_b200.sim import Simulator, default_config  # noqa: E402


def main():
    out_path = sys.argv[1]
    rank, world, local = sdist.init_from_env("nccl")
    data = np.load(os.path.join(os.path.dirname(out_path), "case.npz"))
    cfg = default_config(n_nodes=int(data["n"]), k_indirect=3, fanout=4, pb_cap=6, suspicion_rounds=3, retransmit=5,
                         loss_ppm=int(data["loss"]), seed=int(data["seed"]), rank=rank, world=world, device=local)
    sim = Simulator(cfg)
    sim.set_view(data["nbr"])
    mode = sdist.connect(sim, str(data["mode"]))
    assert mode == str(data["mode"]), f"asked for {data['mode']} exchange, got {mode}"
    sim.inject(np.ascontiguousarray(data["events"]).reshape(-1).view(A.EVENT_DTYPE))
    digests, totals = [], []
    for k, call in enumerate(data["calls"]):
        if data["before"][k]:
            sim.step(int(data["before"][k]))
        args = [data[f"arg{k}_{i}"] for i in range(int(data["nargs"][k]))]
        got = getattr(sim, str(call))(*(a.item() if a.ndim == 0 else a for a in args))
        totals.append([int(v) for v in sdist.global_sum([int(v) for v in np.atleast_1d(got)])])
        for c in data["after"][k]:
            if c:
                sim.step(int(c))
                digests.append(sdist.global_digest(sim.digest()))
    counters = sdist.global_sum(sim.counters())
    mism = int(sdist.global_sum([sim.mismatches()])[0])
    arrays = {A.ARRAY_NAMES[a]: sim.get_array(a) for a in range(A.ARR_COUNT)}
    gathered = [None] * world
    dist.all_gather_object(gathered, arrays)
    if rank == 0:
        REPLICATED = {A.ARRAY_NAMES[a] for a in A.REPLICATED_ARRAYS}
        full = {k: gathered[0][k] if k in REPLICATED else np.concatenate([g[k] for g in gathered]) for k in arrays}
        np.savez(out_path, digests=np.array(digests, dtype=np.uint64), counters=counters, mismatches=mism,
                 totals=np.array([t + [0] * (3 - len(t)) for t in totals], dtype=np.int64), **full)
    dist.barrier()
    sim.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
