"""Time the view generators at 2^20, 2^22 and 2^24 nodes (view_cap = degree = 32): the host generator followed by
swim_sim_set_view, against swim_sim_generate_view (the matrix generated and installed on the device), for the ring,
random and symmetric kinds. Host wall clock around calls that return after the device is done, best of `--reps`; the
two matrices are checked equal once per size and kind. Prints one JSON line with the GPU's name, power limit and
maximum SM clock, and also writes it to the file given with --out. Needs a GPU; not a test.

    python tests/prof_topology.py [--sizes 20,22,24] [--kinds ring,random,symmetric] [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="20,22,24")
    ap.add_argument("--kinds", default="ring,random,symmetric")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    from swim_b200 import _abi as A
    from swim_b200.sim import Simulator, default_config, generate_topology
    out = {"gpu": gpu_info(), "host_threads": len(os.sched_getaffinity(0)), "reps": args.reps,
           "host_generate_s": {}, "host_generate_set_view_s": {}, "generate_view_s": {}, "equal": {}}
    for lg in (int(x) for x in args.sizes.split(",")):
        n = 1 << lg
        with Simulator(default_config(n_nodes=n)) as sim:
            for kind in args.kinds.split(","):
                key = f"{kind} 2^{lg}"
                sim.generate_view(kind, 32, 3)  # warm-up: module load, first allocations
                gen, host, dev = [], [], []
                for _ in range(args.reps):
                    t0 = time.perf_counter()
                    nbr = generate_topology(kind, n, 32, 32, seed=3)
                    t1 = time.perf_counter()
                    sim.set_view(nbr)  # returns after the build has finished on the device
                    t2 = time.perf_counter()
                    gen.append(t1 - t0)
                    host.append(t2 - t0)
                    t0 = time.perf_counter()
                    sim.generate_view(kind, 32, 3)
                    dev.append(time.perf_counter() - t0)
                out["equal"][key] = bool(np.array_equal(sim.get_array(A.ARR_NBR), nbr.reshape(-1)))
                out["host_generate_s"][key] = min(gen)
                out["host_generate_set_view_s"][key] = min(host)
                out["generate_view_s"][key] = min(dev)
                del nbr
                print(key, out["host_generate_set_view_s"][key], out["generate_view_s"][key], out["equal"][key], flush=True)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
