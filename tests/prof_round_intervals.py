"""Per-round view of bench.py's timed window (1 GPU, C3): every round's interval, grouped by class of round.

bench.py reports means over the window. This script runs the same workload, checkpoint, warm-up and launch structure (one
`step` call over the whole window with the in-kernel timeline on) and prints, per class of round:
  * busy rounds: the interval from the round's start to the release of its grid barrier (timeline slots 0 -> 2) as seen
    by CTA 0, and when the slowest CTA arrived at that barrier (slot 5);
  * quiet rounds: the time per round of the batched quiet scans that committed them.
The classes follow the mail load of the C3 trace after the crash at round 10 (heavy at first, tailing off to quiet).

  python tests/prof_round_intervals.py [--steps 448] [--warmup 5] [--json OUT]

Needs a GPU. The card's name and power limit are printed with the numbers: they are part of them.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

CLASSES = [(6, 9), (10, 50), (51, 100), (101, 150), (151, 200), (201, 300), (301, 453)]


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except (OSError, subprocess.SubprocessError):
        import torch
        return {"name": torch.cuda.get_device_name(0), "power.limit": "not read", "clocks.max.sm": "not read"}


def per_round(tl, first_round):
    """[(round, kind, interval_us, slowest_arrival_us)] from the timeline rows; kind 'busy' or 'quiet'. A batched quiet
    scan's rounds share its stamps: each gets the batch time divided by the rounds it committed."""
    out = []
    r = 0
    while r < len(tl):
        t = tl[r]
        rnd = first_round + r
        if t[0] == 0:
            r += 1
            continue
        if t[4] == 0:  # ended after the first barrier: quiet (or a committed batch of quiet rounds)
            span = int(t[7]) if t[7] > 0 else 1
            for q in range(span):
                out.append((rnd + q, "quiet", (t[2] - t[0]) / span / 1e3, None))
            r += span
            continue
        slow = (t[5] - t[0]) / 1e3 if t[5] else None
        end = t[2] if t[3] == 0 else t[4]  # one-barrier rounds end at slot 2, two-barrier rounds at slot 4
        out.append((rnd, "busy", (end - t[0]) / 1e3, slow))
        r += 1
    return out


def summarize(rows):
    res = []
    for lo, hi in CLASSES:
        sel = [x for x in rows if lo <= x[0] <= hi]
        if not sel:
            continue
        busy = [x for x in sel if x[1] == "busy"]
        quiet = [x for x in sel if x[1] == "quiet"]
        iv = np.array([x[2] for x in busy])
        sl = np.array([x[3] for x in busy if x[3] is not None])
        qv = np.array([x[2] for x in quiet])
        res.append({
            "rounds": f"{lo}-{hi}", "busy": len(busy), "quiet": len(quiet),
            "busy_mean_us": float(iv.mean()) if len(iv) else None,
            "busy_median_us": float(np.median(iv)) if len(iv) else None,
            "busy_max_us": float(iv.max()) if len(iv) else None,
            "slowest_cta_arrival_mean_us": float(sl.mean()) if len(sl) else None,
            "quiet_mean_us": float(qv.mean()) if len(qv) else None,
            "total_ms": float(iv.sum() + qv.sum()) / 1e3,
        })
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=448)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", help="also write the result here")
    args = ap.parse_args()

    import bench
    from swim_b200.sim import Simulator, default_config

    cfg_kw, nbr, events, n = bench.workload(1)
    sim = Simulator(default_config(device=0, **cfg_kw))
    sim.set_view(nbr)
    sim.save()
    # clock spin-up as bench.py does, then back to the checkpoint
    sim.load()
    sim.inject(events)
    for _ in range(8):
        sim.step(256)
    sim.load()
    sim.inject(events)
    sim.step(args.warmup)
    sim.set_timeline(args.steps)
    sim.step(args.steps)
    tl = sim.timeline(args.steps).astype(np.int64)
    sim.set_timeline(0)

    rows = per_round(tl, args.warmup + 1)
    out = {"gpu": gpu_info(), "nodes": n, "steps": args.steps, "warmup": args.warmup,
           "window_ms_from_stamps": float(sum(x[2] for x in rows)) / 1e3, "classes": summarize(rows)}
    g = out["gpu"]
    print(f"# {g.get('name')}, power limit {g.get('power.limit')}, max SM clock {g.get('clocks.max.sm')}; "
          f"C3, {n} nodes, rounds {args.warmup + 1}..{args.warmup + args.steps}")
    print(f"{'rounds':>9} {'busy':>5} {'quiet':>5} {'busy mean':>10} {'median':>8} {'max':>8} {'slowest CTA':>12} "
          f"{'quiet mean':>11} {'total ms':>9}")
    fmt = lambda v, w: f"{v:{w}.2f}" if v is not None else f"{'-':>{w}}"
    for c in out["classes"]:
        print(f"{c['rounds']:>9} {c['busy']:5d} {c['quiet']:5d} {fmt(c['busy_mean_us'], 10)} {fmt(c['busy_median_us'], 8)} "
              f"{fmt(c['busy_max_us'], 8)} {fmt(c['slowest_cta_arrival_mean_us'], 12)} {fmt(c['quiet_mean_us'], 11)} "
              f"{c['total_ms']:9.3f}")
    print(f"(times in us; window from the stamps: {out['window_ms_from_stamps']:.3f} ms)")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
