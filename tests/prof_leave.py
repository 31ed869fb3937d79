"""Time graceful leaves at BASELINE config C3's size: one swim_sim_leave of 0.1 % and of 1 % of the nodes, and the
swim_sim_step(1) after it, at 2^20 nodes on 32 slots (random view, D = 32). Host wall clock around calls that return
after a device synchronisation. Prints one JSON line per case and one with everything, including the GPU's name, power
limit and clock read in the same run; --out FILE also writes that line to FILE. Needs a GPU; not a test.

    python tests/prof_leave.py [--nodes-log2 20] [--reps 5] [--out FILE]
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
    ap.add_argument("--nodes-log2", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from swim_b200.sim import Simulator, default_config
    lg = args.nodes_log2
    n = 1 << lg
    out = {"gpu": gpu_info(), "n": f"2^{lg}", "view": "random, D = 32 on 32 slots", "runs": []}
    for frac in (0.001, 0.01):
        rng = np.random.default_rng(lg)
        with Simulator(default_config(n_nodes=n, seed=lg)) as sim:
            sim.generate_view("random", 32, seed=lg)
            sim.step(5)
            sim.leave([0])  # (first call: kernel loads)
            sim.step(1)
            lv, st, res = [], [], []
            for _ in range(args.reps):
                ids = rng.choice(n, size=int(n * frac), replace=False)
                t0 = time.perf_counter()
                res.append(sim.leave(ids))  # returns once the device is done
                lv.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                sim.step(1)
                st.append(time.perf_counter() - t0)
            out["runs"].append({"leavers": int(n * frac), "leave_ms": [round(x * 1e3, 3) for x in lv],
                                "leave_ms_median": round(float(np.median(lv)) * 1e3, 3),
                                "next_step_ms": [round(x * 1e3, 3) for x in st], "left_delivered": res})
        print(json.dumps(out["runs"][-1]), flush=True)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
