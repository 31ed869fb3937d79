"""Bulk membership edits and the device-built mail graph on the SIMT emulator (tests/emu), against the oracle round by
round: swim_sim_set_view_device, swim_sim_remove_dead_nodes and swim_sim_add_members. The H100 versions of these
scenarios are in test_gpu_view_edits.py."""
import numpy as np
import pytest

import view_edit_scenarios as S
from helpers import run_sharded
from swim_b200 import _abi as A
from emu_fixtures import emu_library  # noqa: F401  (autouse fixtures)


@pytest.mark.parametrize("cap", [32, 64, 128, 256])
@pytest.mark.parametrize("kind", ["ring", "random"])
def test_set_view_device_equals_set_view(cap, kind):
    S.set_view_device_equals_set_view(150, cap, kind, min(cap - 4, 40), rounds=6, seed=cap)


@pytest.mark.parametrize("case", ["complete", "hub", "one_node", "vacant_rows", "all_vacant"])
def test_set_view_device_special_graphs(case):
    if case == "complete":
        S.set_view_device_equals_set_view(33, 32, "complete", 32, rounds=6)
    elif case == "hub":  # a member listed by every other node: in-degree N - 1
        S.set_view_device_equals_set_view(700, 32, "random", 20, rounds=5, hub=123)
    elif case == "one_node":
        S.set_view_device_equals_set_view(1, 32, "empty", 0, rounds=3)
    elif case == "vacant_rows":
        S.set_view_device_equals_set_view(200, 64, "random", 30, rounds=5, vacant_rows=40)
    else:
        S.set_view_device_equals_set_view(50, 32, "empty", 0, rounds=3)


def test_set_view_device_validates_like_set_view():
    from swim_b200._lib import SwimError
    from swim_b200.sim import Simulator
    n = 40
    nbr = S.generate_topology("random", n, 32, 10, seed=2)
    for bad, where in ((lambda m: m.__setitem__((7, 3), 7), "row 7 slot 3"),           # self
                       (lambda m: m.__setitem__((9, 2), m[9, 1]), "row 9 slot 2"),     # not ascending
                       (lambda m: m.__setitem__((3, 0), A.NO_MEMBER), "row 3 slot 1"),  # vacancy before a member
                       (lambda m: m.__setitem__((5, 30), n + 2), "row 5 slot 30")):    # id >= N
        m = nbr.copy()
        bad(m)
        for how in ("host", "device"):
            sim = Simulator(S.default_config(n_nodes=n))
            with pytest.raises(SwimError) as e:
                sim.set_view(m) if how == "host" else S.set_view_device(sim, m)
            assert e.value.code == A.EINVAL and where in str(e.value), (how, str(e.value))
            sim.close()
    # rows of other shards are only range-checked
    m = nbr.copy()
    m[35, 4] = n + 1
    sim = Simulator(S.default_config(n_nodes=n, world=2, rank=0))
    with pytest.raises(SwimError) as e:
        S.set_view_device(sim, m)
    assert e.value.code == A.EINVAL and f"entry {35 * 32 + 4} holds id {n + 1}" in str(e.value)
    m[35, 4], m[36, 1] = 36, 35  # a self entry and a non-ascending row in shard 1: shard 0 accepts them
    m[35].sort()
    S.set_view_device(sim, m)
    sim.close()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_set_view_device(world, monkeypatch):
    from swim_b200.sim import Simulator
    monkeypatch.setattr(Simulator, "set_view", S.set_view_device)
    monkeypatch.setenv("SWIM_ROUND_KERNEL", "1")
    run_sharded(world, n=301, chunks=[1] * 4 + [8], loss=20000, deg=24)


@pytest.mark.parametrize("flags,churn,loss", [(0, None, 0), (A.F_STRICT_OVERRIDE | A.F_ROUND_ROBIN, None, 30000),
                                              (A.F_STRICT_OVERRIDE, (20000, 3, 8), 20000)])
def test_remove_dead_nodes_equals_oracle(flags, churn, loss):
    S.remove_dead_then_step(240, 24, before=20, after=15, flags=flags, loss=loss, churn=churn)


@pytest.mark.parametrize("min_age", [1, 7])
def test_remove_dead_nodes_min_age(min_age):
    S.remove_dead_min_age(300, min_age)


def test_add_members_equals_oracle():
    S.add_members_then_step(260, 26, n_adds=120, after=10)


def test_add_members_wide_rows():
    from swim_b200.sim import Simulator
    from oracle.oracle import Oracle
    n, cap = 200, 128
    cfg = S.default_config(n_nodes=n, view_cap=cap, seed=12)
    nbr = S.generate_topology("random", n, cap, 60, seed=12)
    sim, orc = Simulator(cfg), Oracle(cfg)
    sim.set_view(nbr)
    orc.set_view(nbr)
    rng = np.random.default_rng(12)
    obs = rng.integers(0, n, size=300)
    mem = (obs + rng.integers(1, n, size=300)) % n
    inc = rng.integers(0, 9, size=300)
    assert sim.add_members(obs, mem, inc) == S.oracle_add(orc, obs, mem, inc)
    for r in range(4):
        sim.step(1)
        orc.step(1)
        S.assert_same_state(sim, orc, f"round {r + 1}")


def test_error_paths():
    S.error_paths(120)
