"""Time the device-built mail graph: swim_sim_set_view at 2^20, 2^22 and 2^24 nodes (view_cap = degree = 32, host matrix
uploaded), swim_sim_set_view_device at the same sizes (matrix already on the GPU), and at BASELINE config C3 a bulk reap
(swim_sim_remove_dead_nodes after the crash burst) plus the first step after it, which rebuilds the graph. Prints one JSON
line with the GPU's name and power limit. Needs a GPU; not a test.

    python tests/prof_view_build.py [--sizes 20,22,24] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="20,22,24")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    from swim_b200 import _abi as A
    from swim_b200.sim import Simulator, crash_events, default_config, generate_topology
    out = {"gpu": gpu_info(), "set_view_s": {}, "set_view_device_s": {}}
    for lg in (int(x) for x in args.sizes.split(",")):
        n = 1 << lg
        nbr = generate_topology("random", n, 32, 32, seed=3)
        t = torch.from_numpy(nbr.view(np.int32)).cuda()
        with Simulator(default_config(n_nodes=n)) as sim:
            sim.set_view(nbr)  # warm-up: module load, first allocations
            host, dev = [], []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                sim.set_view(nbr)  # returns after the build has finished on the device
                host.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                sim.set_view(t)
                dev.append(time.perf_counter() - t0)
        out["set_view_s"][f"2^{lg}"] = min(host)
        out["set_view_device_s"][f"2^{lg}"] = min(dev)
        del t
        torch.cuda.empty_cache()
    # C3: 1,048 crashes at round 10 of 2^20 nodes, reaped at round 40
    n = 1 << 20
    rng = np.random.default_rng(3)
    with Simulator(default_config(n_nodes=n, seed=0x5EED0001 + 3)) as sim:
        sim.set_view(generate_topology("random", n, 32, 32, seed=3))
        sim.inject(crash_events(10, np.sort(rng.choice(n, size=n // 1000, replace=False)).astype(np.uint32)))
        sim.step(40)
        t0 = time.perf_counter()
        removed = sim.remove_dead_nodes()
        t1 = time.perf_counter()
        sim.step(1)
        t2 = time.perf_counter()
        sim.step(1)
        t3 = time.perf_counter()
    out["c3_reap"] = {"removed": removed, "remove_dead_nodes_s": t1 - t0, "first_step_after_s": t2 - t1,
                      "next_step_s": t3 - t2, "round": 42}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
