"""Time the sharded collectives between steps on ONE device: a world-2 swim_sim_push_pull (both ranks, one host thread
each) and the step after it that rebuilds the mail graph (swim_sim_step(0): the rebuild alone, no round — every rank's
round kernel would need the whole device), against one shard of the same N. Views of 32 slots with 16 members, so the
exchange inserts. Prints one JSON line per size and one with the GPU's name and power limit. Needs a GPU; not a test.

    python tests/prof_sharded_edits.py [--sizes 20,22] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def on_all(sims, fn):
    ts = [threading.Thread(target=fn, args=(s,)) for s in sims]
    t0 = time.perf_counter()
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="20,22")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from swim_b200.sim import Simulator, default_config, generate_topology
    out = {"gpu": gpu_info(), "runs": []}
    for lg in (int(x) for x in args.sizes.split(",")):
        n = 1 << lg
        nbr = generate_topology("random", n, 32, 16, seed=lg)
        row = {"n": f"2^{lg}"}
        for world in (1, 2):
            sims = [Simulator(default_config(n_nodes=n, seed=lg, world=world, rank=r, device=0)) for r in range(world)]
            for s in sims:
                s.set_view(nbr)
            if world > 1:
                blobs = [s.ipc_export() for s in sims]
                for s in sims:
                    s.ipc_connect(blobs)
            pp, rb, res = [], [], []
            for _ in range(args.reps):
                got = [None] * world
                pp.append(on_all(sims, lambda s: got.__setitem__(s.cfg.rank, s.push_pull())))
                res.append([sum(g[k] for g in got) for k in range(3)])
                rb.append(on_all(sims, lambda s: s.step(0)))
            row[f"world{world}"] = {"push_pull_ms": [round(x * 1e3, 2) for x in pp],
                                    "rebuild_step_ms": [round(x * 1e3, 2) for x in rb],
                                    "exchanges_inserted_full": res}
            for s in sims:
                s.close()
        out["runs"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
