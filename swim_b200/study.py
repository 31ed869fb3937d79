"""Convergence-study measurements on top of the bulk simulator (BASELINE config C5: detection latency, false
positives and convergence against the suspicion timeout S). Pure host code over the arrays a handle exposes
(`get_array`, `counters`, `mismatches`): it works on any object with the Simulator's interface.

Terms, per view entry (observer i, member m) of a live observer:
  member down: `detected` = the entry is Dead and was set at or after the crash (latency = vlast - crash round);
               `stale_dead` = Dead since before the crash (an earlier death whose rejoin never reached i);
               otherwise `undetected` (still Alive or Suspect);
  member up:   `suspected` = Suspect (a transient false alarm, or a rejoin that is not known yet);
               `false_dead` = Dead and set after the member's last (re)start — declared dead while it was up;
               `stale_dead_up` = Dead since before the member's last rejoin (the Alive(inc+1) has not arrived).
The mismatch count of the library (`swim_sim_mismatches`) counts every entry that disagrees with the truth, i.e.
undetected + suspected + false_dead + stale_dead_up (a Dead entry of a down member agrees, stale or not).
With graceful leaves (Simulator.leave) a down member that left is not a crash: its entries are `left_entries`, split
into `left_detected` (Dead, set at or after the leave; latency = vlast - leave round) and `left_undetected` (still Alive
or Suspect), and the mismatch count is undetected + suspected + false_dead + stale_dead_up + left_undetected."""
import time

import numpy as np

from . import _abi as A


def event_history(events, n_nodes, upto_round):
    """(last_crash, last_rejoin): the round of each node's last CRASH / REJOIN event with round <= upto_round (0 = none)."""
    last_crash = np.zeros(n_nodes, dtype=np.int64)
    last_rejoin = np.zeros(n_nodes, dtype=np.int64)
    if len(events):
        ev = events[events["round"] <= upto_round]
        order = np.argsort(ev["round"], kind="stable")
        ev = ev[order]
        c = ev[ev["kind"] == A.EV_CRASH]
        last_crash[c["node"]] = c["round"]        # later rounds overwrite earlier ones (sorted ascending)
        r = ev[ev["kind"] == A.EV_REJOIN]
        last_rejoin[r["node"]] = r["round"]
    return last_crash, last_rejoin


def view_report(sim, events, round_now, max_latency=256, left=None):
    """Classify every view entry of this rank's live observers (see the module docstring). Returns a dict of counts
    plus `latency_hist` (index = rounds from crash to the Dead mark, clipped to max_latency). events = None: the crash /
    rejoin rounds come from the handle's SWIM_ARR_LAST_CRASH / SWIM_ARR_LAST_REJOIN arrays (seeded device-side churn).
    left = a bool mask [N] of the processes that left (Simulator.leave): those of them that are down leave the crash
    categories for left_entries / left_detected / left_undetected, and `leave_latency_hist` is returned as well."""
    cap = sim.cfg.view_cap
    alive = sim.get_array(A.ARR_ALIVE).astype(bool)                  # [N] truth, replicated on every rank
    n_total = alive.shape[0]
    nbr = sim.get_array(A.ARR_NBR).reshape(-1, cap)
    st = (sim.get_array(A.ARR_VST).reshape(-1, cap) & 3)
    vlast = sim.get_array(A.ARR_VLAST).reshape(-1, cap).astype(np.int64)
    first = getattr(sim, "first", 0)
    n_local = nbr.shape[0]
    if events is None:  # the library keeps the transition rounds itself (device-side churn has no host trace)
        last_crash = sim.get_array(A.ARR_LAST_CRASH).astype(np.int64)
        last_rejoin = sim.get_array(A.ARR_LAST_REJOIN).astype(np.int64)
    else:
        last_crash, last_rejoin = event_history(events, n_total, round_now)
    observer_up = alive[first:first + n_local][:, None]
    occupied = (st != A.VACANT) & observer_up
    member = np.where(occupied, nbr, 0).astype(np.int64)
    m_up = alive[member]
    down = occupied & ~m_up
    if left is not None:
        gone = down & np.asarray(left, dtype=bool)[member]
        down &= ~gone
    up = occupied & m_up
    dead = st == A.DEAD
    crash_at = last_crash[member]
    detected = down & dead & (vlast >= crash_at)
    lat = np.clip((vlast - crash_at)[detected], 0, max_latency)
    out = {
        "entries": int(occupied.sum()),
        "down_entries": int(down.sum()),
        "detected": int(detected.sum()),
        "stale_dead": int((down & dead & (vlast < crash_at)).sum()),
        "undetected": int((down & ~dead).sum()),
        "suspected": int((up & (st == A.SUSPECT)).sum()),
        "false_dead": int((up & dead & (vlast > last_rejoin[member])).sum()),
        "stale_dead_up": int((up & dead & (vlast <= last_rejoin[member])).sum()),
        "latency_hist": np.bincount(lat, minlength=max_latency + 1).astype(np.int64),
    }
    out["mismatches"] = out["undetected"] + out["suspected"] + out["false_dead"] + out["stale_dead_up"]
    if left is not None:  # (a leave marks the leaver's last_crash: the leave round)
        left_det = gone & dead & (vlast >= crash_at)
        out["left_entries"] = int(gone.sum())
        out["left_detected"] = int(left_det.sum())
        out["left_undetected"] = int((gone & ~dead).sum())
        out["leave_latency_hist"] = np.bincount(np.clip((vlast - crash_at)[left_det], 0, max_latency),
                                                minlength=max_latency + 1).astype(np.int64)
        out["mismatches"] += out["left_undetected"]
    return out


def merge_reports(reports):
    """Sum per-rank reports (all values are counts)."""
    out = {}
    for r in reports:
        for k, v in r.items():
            out[k] = out[k] + v if k in out else (v.copy() if isinstance(v, np.ndarray) else v)
    return out


def latency_stats(hist):
    """mean / p50 / p99 / max of a latency histogram (None when empty)."""
    total = int(hist.sum())
    if total == 0:
        return {"n": 0, "mean": None, "p50": None, "p99": None, "max": None}
    idx = np.arange(len(hist))
    cum = np.cumsum(hist)
    return {"n": total, "mean": float((idx * hist).sum() / total),
            "p50": int(np.searchsorted(cum, 0.5 * total)), "p99": int(np.searchsorted(cum, 0.99 * total)),
            "max": int(np.flatnonzero(hist)[-1])}


def restart_joins(sim, hosts, since, upto):
    """memberlist's restart, Join(joinHosts): every up process whose last rejoin lies in rounds (since, upto] paired with
    each join host (never with itself). Built from the replicated SWIM_ARR_ALIVE / SWIM_ARR_LAST_REJOIN arrays, so every
    rank builds the same list. Returns (nodes, seeds)."""
    hosts = np.asarray(hosts, dtype=np.uint32)
    alive = sim.get_array(A.ARR_ALIVE).astype(bool)
    back = sim.get_array(A.ARR_LAST_REJOIN).astype(np.int64)
    who = np.flatnonzero(alive & (back > since) & (back <= upto)).astype(np.uint32)
    nodes, seeds = np.repeat(who, len(hosts)), np.tile(hosts, len(who))
    keep = nodes != seeds
    return nodes[keep], seeds[keep]


def leave_draw(sim, seed, round_, leave_ppm):
    """The processes that leave gracefully after round `round_`: each up process with probability leave_ppm / 1e6, drawn
    from a host generator seeded by (seed, round), so every rank, and every suspicion timeout of a sweep, draws the
    same. Returns the ids (ascending)."""
    alive = sim.get_array(A.ARR_ALIVE).astype(bool)
    draw = np.random.default_rng([seed, round_]).random(alive.shape[0]) < leave_ppm * 1e-6
    return np.flatnonzero(alive & draw).astype(np.uint32)


def run_sweep_point(sim, events, rounds, sample_every=10, reduce_sum=None, push_pull_every=0, join_hosts=None,
                    join_fresh=False, leave_ppm=0):
    """Step `rounds` rounds, sampling the convergence count; returns the time series, the final counters and the final
    view report. `reduce_sum(list_of_numbers) -> list` adds values over ranks (identity for one GPU). push_pull_every = R
    > 0: a push-pull state exchange (Simulator.push_pull; on a sharded handle a collective, which every rank reaches at
    the same round) after every R-th round; its outputs, summed over the calls and the ranks, are in "push_pull".
    join_hosts = the ids of K join hosts: after every step chunk the processes that restarted in it join through all K
    (Simulator.join, `fresh` = join_fresh: the restart lost its state; a collective on a sharded handle). The summed
    outputs, the joins and the host time of the calls are in "join". leave_ppm > 0: after every step chunk each up
    process leaves gracefully (Simulator.leave) with probability leave_ppm / 1e6 (leave_draw, seeded by the config's seed
    and the round); the report then counts the left members apart, and "leave" holds the calls, ids listed, leavers,
    records delivered, the host time of the calls and the leave detection latency."""
    red = reduce_sum or (lambda xs: xs)
    series = []
    done = 0
    device_ms = 0.0
    pp = [0, 0, 0]
    jn = [0, 0, 0, 0]  # exchanges, inserted, full, pairs
    join_s = 0.0
    lv = [0, 0, 0, 0]  # calls, listed, left, delivered
    leave_s = 0.0
    left = np.zeros(int(sim.cfg.n_nodes), dtype=bool) if leave_ppm else None
    while done < rounds:
        step = min(sample_every - done % sample_every, rounds - done)
        if push_pull_every:
            step = min(step, push_pull_every - done % push_pull_every)
        sim.step(step)
        if hasattr(sim, "last_step_ms"):
            device_ms += float(sim.last_step_ms())  # CUDA events around the call's kernels, this rank
        done += step
        if join_hosts is not None and len(join_hosts):
            nodes, seeds = restart_joins(sim, join_hosts, done - step, done)
            t0 = time.perf_counter()
            got = sim.join(nodes, seeds, join_fresh)  # (returns after a device synchronisation)
            join_s += time.perf_counter() - t0
            jn = [a + b for a, b in zip(jn, list(got) + [len(nodes)])]
        if leave_ppm:
            ids = leave_draw(sim, int(sim.cfg.seed), int(sim.round), leave_ppm)
            if len(ids):
                t0 = time.perf_counter()
                got = sim.leave(ids)  # (returns after a device synchronisation)
                leave_s += time.perf_counter() - t0
                left[ids] = True
                lv = [a + b for a, b in zip(lv, [1, len(ids)] + list(got))]
        if push_pull_every and done % push_pull_every == 0:
            pp = [a + b for a, b in zip(pp, sim.push_pull())]
        if done % sample_every == 0 or done == rounds:
            series.append((done, int(red([sim.mismatches()])[0])))
    counters = [int(x) for x in red([int(v) for v in sim.counters()])]
    rep = view_report(sim, events, done, left=left)
    hist = np.array(red(rep.pop("latency_hist").tolist()), dtype=np.int64)
    lhist = np.array(red(rep.pop("leave_latency_hist").tolist()), dtype=np.int64) if left is not None else None
    keys = sorted(rep)
    vals = red([rep[k] for k in keys])
    rep = dict(zip(keys, (int(v) for v in vals)))
    rep["latency"] = latency_stats(hist)
    out = {"mismatch_series": series, "counters": dict(zip(A.CTR_NAMES, counters)), "report": rep,
           "device_ms": device_ms, "device_us_per_round": device_ms * 1e3 / max(1, rounds)}
    if push_pull_every:
        out["push_pull"] = dict(zip(("exchanges", "inserted", "full"), (int(v) for v in red(pp))))
    if join_hosts is not None and len(join_hosts):
        out["join"] = dict(zip(("exchanges", "inserted", "full"), (int(v) for v in red(jn[:3]))))
        out["join"].update(pairs=jn[3], host_s_rank0=join_s)
    if leave_ppm:
        out["leave"] = dict(calls=lv[0], listed=lv[1], left=int(red([lv[2]])[0]), delivered=int(red([lv[3]])[0]),
                            host_s_rank0=leave_s, leave_latency=latency_stats(lhist))
    return out
