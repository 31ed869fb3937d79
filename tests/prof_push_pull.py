"""Time the push-pull state exchange: one swim_sim_push_pull call, and the swim_sim_step(1) after it (which rebuilds the
mail graph when the call inserted members), at 2^20, 2^22 and 2^24 nodes on 32 slots, with full rows (D = 32: no
inserts) and half-full rows (D = 16: inserts). Prints one JSON line with the GPU's name and power limit. Needs a GPU;
not a test.

    python tests/prof_push_pull.py [--sizes 20,22,24] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

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
    from swim_b200.sim import Simulator, default_config, generate_topology
    out = {"gpu": gpu_info(), "runs": []}
    for lg in (int(x) for x in args.sizes.split(",")):
        n = 1 << lg
        for deg in (32, 16):
            with Simulator(default_config(n_nodes=n, seed=lg)) as sim:
                sim.set_view(generate_topology("random", n, 32, deg, seed=lg))
                sim.step(5)
                pp, st, res = [], [], []
                for _ in range(args.reps):
                    t0 = time.perf_counter()
                    res.append(sim.push_pull())  # returns once the device is done
                    pp.append(time.perf_counter() - t0)
                    t0 = time.perf_counter()
                    sim.step(1)
                    st.append(time.perf_counter() - t0)
                out["runs"].append({"n": f"2^{lg}", "degree": deg, "push_pull_ms": [round(x * 1e3, 2) for x in pp],
                                    "next_step_ms": [round(x * 1e3, 2) for x in st],
                                    "exchanges_inserted_full": res})
            print(json.dumps(out["runs"][-1]), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
