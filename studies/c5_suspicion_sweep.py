#!/usr/bin/env python
"""BASELINE config C5 — churn and a suspicion-timeout sweep (SURVEY 8(d)): detection latency, false positives and
convergence against S, on 1..8 GPUs.

    python studies/c5_suspicion_sweep.py --nodes-per-gpu 65536 --rounds 300
    torchrun --nproc-per-node 8 studies/c5_suspicion_sweep.py --nodes-per-gpu 2097152 --rounds 1000   # C5 itself

The churn is generated ON THE DEVICE (cfg.churn_ppm: every round each live process crashes with probability crash_ppm / 1e6
and rejoins after U[10, 50] rounds with incarnation + 1 and an Alive broadcast; Philox purpose 7, mirrored by the oracle).
ONE handle serves the whole sweep: the view and its in-edge index are built once, swim_sim_save keeps round 0 on the device,
and every S is swim_sim_load + swim_sim_set_params(suspicion_rounds = S). One JSON line per S on rank 0:
  detection latency (rounds from the crash to the observer's Dead mark: mean / p50 / p99 / max over all entries whose
  member is down at the end), undetected / stale entries, false positives (entries Dead while the member was up;
  refutations), the mismatch time series, device time per round.
The CUDA library does the stepping; this file and swim_b200/study.py only read arrays back."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
# torchrun exports OMP_NUM_THREADS=1 to its workers; the host-side index build (swim_sim_set_view) is OpenMP code
_w = max(1, int(os.environ.get("LOCAL_WORLD_SIZE", os.environ.get("WORLD_SIZE", "1"))))
os.environ["OMP_NUM_THREADS"] = str(max(1, len(os.sched_getaffinity(0)) // _w))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes-per-gpu", type=int, default=65536)
    ap.add_argument("--rounds", type=int, default=300)
    ap.add_argument("--suspicion", type=int, nargs="+", default=[2, 3, 5, 8, 13])
    ap.add_argument("--suspicion-max", type=int, default=0, help="Lifeguard-style dynamic timeout: start value (0 = off)")
    ap.add_argument("--crash-ppm", type=int, default=1000)
    ap.add_argument("--loss-ppm", type=int, default=0)
    ap.add_argument("--flags", type=int, default=0, help="SWIM_F_* protocol variants")
    ap.add_argument("--topology", default="random", choices=["random", "ring", "symmetric"],
                    help="view graph, generated on the device: directed random views, a ring lattice, or symmetric random "
                         "views (j lists i exactly when i lists j)")
    ap.add_argument("--sample-every", type=int, default=10)
    ap.add_argument("--push-pull-every", type=int, default=0, metavar="R",
                    help="a push-pull state exchange (memberlist anti-entropy) after every R-th round (a collective "
                         "on several GPUs)")
    ap.add_argument("--join-hosts", type=int, default=0, metavar="K",
                    help="K join hosts drawn once from the seed: after every step chunk each process that restarted in "
                         "it joins through all K (memberlist's Join(joinHosts); a collective on several GPUs)")
    ap.add_argument("--join-fresh", action="store_true",
                    help="the restarted processes lose their view and piggyback buffer before joining")
    ap.add_argument("--leave-ppm", type=int, default=0, metavar="P",
                    help="after every step chunk each up process leaves gracefully (memberlist's Leave) with "
                         "probability P / 10^6, the same draw on every rank and for every S (a collective on several GPUs)")
    ap.add_argument("--seed", type=int, default=0x5EED0001 + 5)
    args = ap.parse_args()

    import torch
    from swim_b200 import dist as sd
    from swim_b200.sim import Simulator, default_config
    from swim_b200.study import run_sweep_point

    rank, world, local = sd.init_from_env()
    if not torch.cuda.is_available():
        raise SystemExit("c5_suspicion_sweep needs a CUDA device (there is no CPU fallback)")
    torch.cuda.set_device(local)
    n = args.nodes_per_gpu * world
    red = (lambda xs: [int(v) for v in sd.global_sum(xs)]) if world > 1 else None

    def barrier():
        torch.cuda.synchronize()  # never an NCCL kernel next to a sharded round kernel in flight (DESIGN.md section 9)
        if world > 1:
            import torch.distributed as dist
            dist.barrier()
            torch.cuda.synchronize()

    cfg = default_config(n_nodes=n, suspicion_rounds=args.suspicion[0], loss_ppm=args.loss_ppm, seed=args.seed, rank=rank,
                         world=world, device=local, flags=args.flags, churn_ppm=args.crash_ppm, rejoin_min=10, rejoin_max=50)
    def setup():
        t0 = time.perf_counter()
        sim = Simulator(cfg)
        t1 = time.perf_counter()
        sim.generate_view(args.topology, 32, seed=args.seed & 0xFFFF)  # every rank generates the global matrix on its GPU
        t_topo = time.perf_counter() - t1
        mode = sd.connect(sim)
        sim.save()
        return sim, mode, t_topo, time.perf_counter() - t0 - t_topo

    sim, mode, t_topo, t_setup = setup()
    hosts = None
    if args.join_hosts:  # the same draw on every rank
        import numpy as np
        hosts = np.sort(np.random.default_rng(args.seed).choice(n, size=args.join_hosts, replace=False)).astype(np.uint32)
    for k, S in enumerate(args.suspicion):
        barrier()
        if k and args.join_hosts:  # a join that changed memberships dropped the checkpoint
            sim.close()
            sim, mode, t_topo, t_setup = setup()
        sim.load()
        smax = max(args.suspicion_max, S) if args.suspicion_max else 0
        sim.set_params(suspicion_rounds=S, suspicion_max=min(smax, 15))
        barrier()
        t0 = time.perf_counter()
        res = run_sweep_point(sim, None, args.rounds, args.sample_every, red, args.push_pull_every, hosts,
                              args.join_fresh, args.leave_ppm)
        wall = time.perf_counter() - t0
        if rank == 0:
            rep = res["report"]
            line = {"config": {"workload": "C5", "n_nodes": n, "n_gpus": world, "rounds": args.rounds, "S": S,
                               "suspicion_max": min(smax, 15), "crash_ppm": args.crash_ppm, "loss_ppm": args.loss_ppm,
                               "flags": args.flags, "exchange": mode, "topology": args.topology,
                               "churn": "device-side, Philox purpose 7, rejoin U[10,50]"},
                    "detection_latency_rounds": rep.pop("latency"),
                    "entries": rep, "counters": res["counters"],
                    "false_positive_rate": (rep["false_dead"] + res["counters"]["refutes"]) / max(1, res["counters"]["pings"]),
                    "mismatch_series": res["mismatch_series"], "wall_s": wall,
                    "device_us_per_round_rank0": res["device_us_per_round"],
                    "node_rounds_per_s_device_rank0": n * args.rounds / max(1e-9, res["device_ms"] * 1e-3),
                    "node_rounds_per_s_wall": n * args.rounds / wall,
                    "setup_s": {"topology": t_topo, "create_connect_save": t_setup}}
            if args.push_pull_every:
                line["config"]["push_pull_every"] = args.push_pull_every
                line["push_pull"] = res["push_pull"]
            if args.join_hosts:
                line["config"].update(join_hosts=hosts.tolist(), join_fresh=args.join_fresh)
                line["join"] = res["join"]
            if args.leave_ppm:
                line["config"]["leave_ppm"] = args.leave_ppm
                line["leave"] = res["leave"]
            print(json.dumps(line), flush=True)
    sim.close()
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
