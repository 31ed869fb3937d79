"""Time seed joins: one swim_sim_join of 1 % of the nodes, each through the same 3 join hosts, and the swim_sim_step(1)
after it (which rebuilds the mail graph when the join changed memberships), at 2^20, 2^22 and 2^24 nodes on 32 slots
(random views, D = 32), with and without SWIM_JOIN_FRESH. Host wall clock around calls that return after a device
synchronisation. Prints one JSON line per case and one with everything, including the GPU's name and power limit read in
the same run; --out FILE also writes that line to FILE. Needs a GPU; not a test.

    python tests/prof_join.py [--sizes 20,22,24] [--reps 3] [--out FILE]
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
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from swim_b200.sim import Simulator, default_config
    out = {"gpu": gpu_info(), "runs": []}
    for lg in (int(x) for x in args.sizes.split(",")):
        n = 1 << lg
        rng = np.random.default_rng(lg)
        hosts = rng.choice(n, size=3, replace=False)
        for fresh in (False, True):
            with Simulator(default_config(n_nodes=n, seed=lg)) as sim:
                sim.generate_view("random", 32, seed=lg)
                sim.step(5)
                jn, st, res = [], [], []
                for _ in range(args.reps):
                    who = rng.choice(n, size=n // 100, replace=False)
                    nodes, seeds = np.repeat(who, 3), np.tile(hosts, len(who))
                    keep = nodes != seeds
                    t0 = time.perf_counter()
                    res.append(sim.join(nodes[keep], seeds[keep], fresh))  # returns once the device is done
                    jn.append(time.perf_counter() - t0)
                    t0 = time.perf_counter()
                    sim.step(1)
                    st.append(time.perf_counter() - t0)
                out["runs"].append({"n": f"2^{lg}", "fresh": fresh, "pairs": int(keep.sum()),
                                    "join_ms": [round(x * 1e3, 2) for x in jn],
                                    "next_step_ms": [round(x * 1e3, 2) for x in st],
                                    "exchanges_inserted_full": res})
            print(json.dumps(out["runs"][-1]), flush=True)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
