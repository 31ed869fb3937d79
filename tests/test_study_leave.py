"""The convergence study with graceful leaves (swim_b200/study.py): view_report(left=...) against a plain restatement
of its terms, entry by entry; the mismatch identity undetected + suspected + false_dead + stale_dead_up + left_undetected
= swim_sim_mismatches; the default report unchanged by the new argument; and run_sweep_point(leave_ppm=...) on the
device code (the SIMT emulator) against the oracle."""
import os

import numpy as np
import pytest

from between_steps_oracle import leave as oracle_leave
from oracle.oracle import Oracle
from swim_b200 import _abi as A
from swim_b200.sim import default_config, generate_topology
from swim_b200.study import run_sweep_point, view_report

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class LeavingOracle(Oracle):
    def leave(self, ids):
        return oracle_leave(self, ids)


def churned(n=240, seed=31, rounds=30, leave_every=6, frac=0.03):
    """An oracle under seeded churn and loss, with a leave of `frac` of the nodes every `leave_every` rounds. Returns it
    and the bool mask of the processes that left."""
    cfg = default_config(n_nodes=n, seed=seed, suspicion_rounds=4, loss_ppm=20000, churn_ppm=15000, rejoin_min=3,
                         rejoin_max=9)
    orc = LeavingOracle(cfg)
    orc.set_view(generate_topology("random", n, 32, 12, seed=seed))
    rng = np.random.default_rng(seed)
    left = np.zeros(n, dtype=bool)
    for _ in range(rounds // leave_every):
        orc.step(leave_every)
        ids = rng.choice(n, size=int(n * frac), replace=False)
        left[ids[orc.get_array(A.ARR_ALIVE)[ids] != 0]] = True  # (a down id is not a leaver)
        orc.leave(ids)
    orc.step(3)
    return orc, left


def restated(orc, left):
    """view_report's terms, one view entry at a time."""
    n, cap = orc.cfg.n_nodes, orc.cfg.view_cap
    alive = orc.get_array(A.ARR_ALIVE)
    nbr, st = orc.get_array(A.ARR_NBR).reshape(n, cap), orc.get_array(A.ARR_VST).reshape(n, cap) & 3
    vlast = orc.get_array(A.ARR_VLAST).reshape(n, cap)
    crash, rejoin = orc.get_array(A.ARR_LAST_CRASH), orc.get_array(A.ARR_LAST_REJOIN)
    keys = ("entries", "down_entries", "detected", "stale_dead", "undetected", "suspected", "false_dead", "stale_dead_up",
            "left_entries", "left_detected", "left_undetected")
    out = dict.fromkeys(keys, 0)
    lat, llat = [], []
    for i in range(n):
        if not alive[i]:
            continue
        for s in range(cap):
            if st[i, s] == A.VACANT:
                continue
            m, dead, v = int(nbr[i, s]), st[i, s] == A.DEAD, int(vlast[i, s])
            out["entries"] += 1
            if alive[m]:
                out["suspected"] += st[i, s] == A.SUSPECT
                out["false_dead"] += dead and v > rejoin[m]
                out["stale_dead_up"] += dead and v <= rejoin[m]
            elif left[m]:
                out["left_entries"] += 1
                out["left_detected"] += dead and v >= crash[m]
                out["left_undetected"] += not dead
                if dead and v >= crash[m]:
                    llat.append(v - int(crash[m]))
            else:
                out["down_entries"] += 1
                out["detected"] += dead and v >= crash[m]
                out["stale_dead"] += dead and v < crash[m]
                out["undetected"] += not dead
                if dead and v >= crash[m]:
                    lat.append(v - int(crash[m]))
    return out, lat, llat


def test_view_report_with_left_members():
    orc, left = churned()
    rep = view_report(orc, None, orc.round, left=left)
    want, lat, llat = restated(orc, left)
    for k, v in want.items():
        assert rep[k] == v, (k, rep[k], v)
    assert rep["left_entries"] > 0 and rep["left_detected"] > 0 and rep["detected"] > 0
    assert np.array_equal(rep["latency_hist"], np.bincount(lat, minlength=257))
    assert np.array_equal(rep["leave_latency_hist"], np.bincount(llat, minlength=257))
    ident = rep["undetected"] + rep["suspected"] + rep["false_dead"] + rep["stale_dead_up"] + rep["left_undetected"]
    assert rep["mismatches"] == ident == orc.mismatches()


def test_default_report_is_unchanged():
    orc, _ = churned(n=160, seed=32)
    rep = view_report(orc, None, orc.round)
    assert not any(k.startswith("left") or k.startswith("leave") for k in rep)
    base = view_report(orc, None, orc.round, left=np.zeros(160, dtype=bool))
    for k, v in rep.items():
        if k != "latency_hist":
            assert base[k] == v, k
    assert base["left_entries"] == 0


@pytest.fixture
def emu_library(monkeypatch):
    import sys
    import swim_b200._lib as L
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu
    so = build_emu.build()
    saved = (L.SO_PATH, L._lib)
    L.SO_PATH, L._lib = so, None
    assert L.lib().swim_abi_version() == A.ABI_VERSION
    yield
    L.SO_PATH, L._lib = saved


@pytest.mark.usefixtures("emu_library")
def test_sweep_point_with_leaves_matches_oracle():
    """run_sweep_point with leave_ppm under seeded churn: the same draws, series, counters, report and leave totals on
    the device code and on the oracle."""
    from swim_b200.sim import Simulator
    n = 300
    cfg = default_config(n_nodes=n, seed=21, suspicion_rounds=3, churn_ppm=20000, rejoin_min=3, rejoin_max=8)
    nbr = generate_topology("random", n, 32, 12, seed=21)
    out = []
    for h in (Simulator(cfg), LeavingOracle(cfg)):
        h.set_view(nbr)
        res = run_sweep_point(h, None, 40, 10, leave_ppm=20000)
        res["leave"].pop("host_s_rank0")
        out.append({k: res[k] for k in ("mismatch_series", "counters", "report", "leave")})
    assert out[0] == out[1]
    lv, rep = out[0]["leave"], out[0]["report"]
    assert lv["calls"] > 0 and lv["left"] > 0 and lv["delivered"] > 0 and lv["leave_latency"]["n"] > 0
    assert rep["left_entries"] > 0
