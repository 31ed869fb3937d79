"""Seed joins (swim_sim_join) on the H100, against the oracle: the shared scenarios at 2^16 nodes for every row width,
BASELINE config C3 (2^20 nodes, crash burst) with joins every 25 rounds, a 2^20-node fresh join that forces the graph
rebuild, and sharded handles of world 2 and 4 on one device. The emulator versions are in test_emu_join.py."""
import numpy as np
import pytest

import join_scenarios as S
from helpers import crash_events, default_config, generate_topology, make_pair
from between_steps_oracle import join as oracle_join
from nccl_fixtures import fake_nccl_gpu, fake_nccl_gpu_lib, staged_too  # noqa: F401  (fixtures)
from swim_b200 import _abi as A

pytestmark = pytest.mark.gpu
N16 = 1 << 16


@pytest.fixture
def fused_exchange(monkeypatch):
    monkeypatch.setenv("SWIM_ROUND_KERNEL", "1")


@pytest.mark.parametrize("cap", [32, 64, 128, 256])
def test_every_row_width(cap):
    S.join_every(N16, cap, cap - 8, rounds=18, every=6, seed=cap, loss_ppm=20000, churn_ppm=2000, rejoin_min=2,
                 rejoin_max=6)


@pytest.mark.parametrize("flags,suspicion_max", [(A.F_STRICT_OVERRIDE, 0), (0, 9)])
def test_protocol_variants(flags, suspicion_max):
    S.join_every(N16, 32, 20, rounds=30, every=5, flags=flags, suspicion_max=suspicion_max, loss_ppm=20000)


def test_hub():
    S.hub(N16, 5000)


def test_save_join_load():
    S.save_join_load(N16)


def test_with_push_pull():
    S.with_push_pull(N16)


def test_error_paths():
    S.error_paths(N16)


def test_c3_joins_every_25_rounds():
    """C3: N = 1,048,576, D = 32 on 32 slots, 1,048 crashes at round 10; every 25 rounds the crashed nodes' ids join
    through 3 fixed seeds (they are down, so only the seeds' other pairs exchange) together with 0.1 % random up nodes,
    over 200 rounds."""
    n = 1 << 20
    cfg = default_config(n_nodes=n, seed=0x5EED0001 + 3)
    rng = np.random.default_rng(3)
    crashed = np.sort(rng.choice(n, size=n // 1000, replace=False)).astype(np.uint32)
    sim, orc = make_pair(cfg, generate_topology("random", n, 32, 32, seed=3))
    ev = crash_events(10, crashed)
    sim.inject(ev)
    orc.inject(ev)
    hosts = rng.choice(n, size=3, replace=False)
    for k in range(8):
        sim.step(25)
        orc.step(25)
        nodes, seeds = S.restart_pairs(rng, n, hosts, frac=0.001)
        nodes, seeds = np.concatenate([nodes, crashed[:30]]), np.concatenate([seeds, np.full(30, hosts[0])])
        keep = nodes != seeds
        got = sim.join(nodes[keep], seeds[keep], fresh=k % 2 == 1)
        assert got == oracle_join(orc, nodes[keep], seeds[keep], fresh=k % 2 == 1), got
        assert sim.digest() == orc.digest(), f"digest differs at round {sim.round}"
        assert sim.counters().tolist() == orc.counters().tolist()
    sim.step(5)
    orc.step(5)
    assert sim.digest() == orc.digest() and sim.mismatches() == orc.mismatches()
    sim.close()


def test_fresh_join_forces_rebuild():
    S.fresh_rebuild(1 << 20, frac=0.01, hosts=3, deg=16, rounds=(1, 9, 40))


@pytest.mark.usefixtures("fused_exchange")
@pytest.mark.parametrize("world,mode", staged_too([2, 4], ["2", "4"]))
def test_sharded(world, mode, request):
    """Over peer memory, and through the staged exchange with the in-process NCCL stand-in ("nccl")."""
    if mode == "nccl":
        request.getfixturevalue("fake_nccl_gpu")
    S.sharded_joins(world, 1100, mode, devices=[0] * world, rounds=36, every=12)


def test_sharded_equals_single_shard():
    S.sharded_equals_single_shard(1 << 18, 4, [0] * 4)
