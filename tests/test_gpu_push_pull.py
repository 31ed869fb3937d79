"""The push-pull state exchange (swim_sim_push_pull) on the GPU, against the oracle: the shared scenarios at 2^16 nodes,
BASELINE config C3 (2^20 nodes, full rows) with its crash burst and a push_pull every 25 rounds, a 2^20-node random view
with D = 16 of 32 slots (inserts, then the graph rebuild), and a ring."""
import numpy as np
import pytest

import push_pull_scenarios as S
from helpers import crash_events, default_config, generate_topology, make_pair
from between_steps_oracle import push_pull as oracle_push_pull
from swim_b200 import _abi as A

pytestmark = pytest.mark.gpu
N16 = 1 << 16


@pytest.mark.parametrize("cap", [32, 64, 128, 256])
def test_every_row_width(cap):
    S.step_push_pull_step(N16, cap, cap - 8, rounds=18, every=6, seed=cap, loss_ppm=20000)


@pytest.mark.parametrize("flags,suspicion_max", [(A.F_STRICT_OVERRIDE, 0), (0, 9)])
def test_churn_loss_and_variants(flags, suspicion_max):
    S.step_push_pull_step(N16, 32, 20, rounds=30, every=5, flags=flags, suspicion_max=suspicion_max, loss_ppm=20000,
                          churn_ppm=2000, rejoin_min=2, rejoin_max=6)


def test_save_push_pull_load():
    S.save_push_pull_load(N16)


def test_inserts_then_rounds():
    S.inserts_then_rounds(N16, 64, deg=20, rounds=50)


def test_push_pull_then_edits():
    S.push_pull_then_edits(N16)


def test_export_after_push_pull():
    S.export_after_push_pull(1 << 12)


def test_error_paths():
    S.error_paths(N16)


def _digest_equal(sim, orc, where):
    assert sim.digest() == orc.digest(), f"digest differs: {where}"
    assert sim.counters().tolist() == orc.counters().tolist(), f"counters differ: {where}"
    assert sim.mismatches() == orc.mismatches(), f"mismatch count differs: {where}"


def test_c3_push_pull_every_25_rounds():
    """C3: N = 1,048,576, D = 32 on 32 slots (full rows: no inserts), 1,048 crashes at round 10; push_pull every 25
    rounds over 200 rounds."""
    n = 1 << 20
    cfg = default_config(n_nodes=n, seed=0x5EED0001 + 3)
    crashed = np.sort(np.random.default_rng(3).choice(n, size=n // 1000, replace=False)).astype(np.uint32)
    sim, orc = make_pair(cfg, generate_topology("random", n, 32, 32, seed=3))
    ev = crash_events(10, crashed)
    sim.inject(ev)
    orc.inject(ev)
    for _ in range(8):
        sim.step(25)
        orc.step(25)
        got = sim.push_pull()
        assert got == oracle_push_pull(orc) and got[1] == 0
        _digest_equal(sim, orc, f"round {sim.round}")
    sim.close()


def test_random_view_with_inserts():
    """2^20 nodes, D = 16 on 32 slots: push_pull inserts, and the 100 rounds after the rebuild match the oracle."""
    n = 1 << 20
    cfg = default_config(n_nodes=n, seed=17, loss_ppm=10000)
    sim, orc = make_pair(cfg, generate_topology("random", n, 32, 16, seed=17))
    ev = crash_events(3, np.random.default_rng(17).choice(n, size=n // 500, replace=False))
    sim.inject(ev)
    orc.inject(ev)
    sim.step(5)
    orc.step(5)
    got = sim.push_pull()
    assert got == oracle_push_pull(orc) and got[1] > 0, got
    for a in (A.ARR_NBR, A.ARR_VST, A.ARR_VINC, A.ARR_VLAST, A.ARR_PB, A.ARR_SELF_INC):
        assert np.array_equal(sim.get_array(a), orc.get_array(a)), A.ARRAY_NAMES[a]
    for chunk in (1, 9, 40, 50):
        sim.step(chunk)
        orc.step(chunk)
        _digest_equal(sim, orc, f"round {sim.round}")
    sim.close()


def test_ring():
    S.inserts_then_rounds(1 << 18, 32, deg=4, rounds=30, kind="ring", seed=19)
