"""Bulk membership edits and the device-built mail graph on the GPU, against the oracle: swim_sim_set_view_device (torch
int32 / uint32 input, sharded on one device, a hub of in-degree >= 10^5), swim_sim_remove_dead_nodes and
swim_sim_add_members at 2^16 - 2^20 nodes, and BASELINE config C3 reaped after its crash burst."""
import numpy as np
import pytest

import view_edit_scenarios as S
from helpers import crash_events, default_config, generate_topology, make_pair, run_sharded
from swim_b200 import _abi as A

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cap,dtype", [(32, "int32"), (64, "uint32"), (128, "int32"), (256, "uint32")])
def test_set_view_device_equals_set_view(cap, dtype):
    S.set_view_device_equals_set_view(1 << 16, cap, "random", cap - 8, rounds=4, seed=cap, dtype=dtype)


@pytest.mark.parametrize("kind,n,deg", [("ring", 1 << 18, 16), ("complete", 33, 32)])
def test_set_view_device_ring_and_complete(kind, n, deg):
    S.set_view_device_equals_set_view(n, 32, kind, deg, rounds=4)


def test_set_view_device_hub():
    """One member listed by every other node of 2^17: an in-list of 131,071 senders."""
    S.set_view_device_equals_set_view(1 << 17, 32, "random", 16, rounds=3, hub=4242, vacant_rows=100)


def test_set_view_device_rejects_a_tensor_it_cannot_read():
    import torch
    from swim_b200.sim import Simulator
    sim = Simulator(default_config(n_nodes=64))
    for bad in (torch.zeros(64 * 32, dtype=torch.int64, device="cuda"), torch.zeros(64 * 31, dtype=torch.int32, device="cuda"),
                torch.zeros((32, 128), dtype=torch.int32, device="cuda").t()):
        with pytest.raises(ValueError):
            sim.set_view(bad)
    sim.close()


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_set_view_device_one_device(world, monkeypatch):
    """Small shards, as in test_gpu_shards_one_device.py: every rank's kernel must be resident at once on the one GPU."""
    from swim_b200.sim import Simulator
    monkeypatch.setattr(Simulator, "set_view", S.set_view_device)
    run_sharded(world, n=1201, chunks=[1] * 4 + [14, 30], loss=20000, deg=24, devices=[0] * world)


@pytest.mark.parametrize("flags,churn", [(0, None), (A.F_STRICT_OVERRIDE | A.F_ROUND_ROBIN, (5000, 3, 10))])
def test_remove_dead_nodes_equals_oracle(flags, churn):
    S.remove_dead_then_step(1 << 16, 32, before=25, after=20, flags=flags, loss=20000, churn=churn, every_round=False)


def test_remove_dead_nodes_min_age():
    S.remove_dead_min_age(1 << 17, 5)


def test_add_members_equals_oracle():
    S.add_members_then_step(1 << 16, 30, n_adds=20000, after=12, every_round=False)


def test_error_paths():
    S.error_paths(1 << 16)


def test_c3_reap_after_the_burst():
    """BASELINE config C3 (N = 1,048,576, 1,048 crashes at round 10): through the burst, removeDeadNodes on every store,
    then 100 more rounds with digest, counters and convergence count equal to the oracle's."""
    n = 1 << 20
    cfg = default_config(n_nodes=n, seed=0x5EED0001 + 3)
    rng = np.random.default_rng(3)
    crashed = np.sort(rng.choice(n, size=n // 1000, replace=False)).astype(np.uint32)
    sim, orc = make_pair(cfg, generate_topology("random", n, 32, 32, seed=3))
    ev = crash_events(10, crashed)
    sim.inject(ev)
    orc.inject(ev)
    sim.step(40)
    orc.step(40)
    want = S.dead_entries(orc)
    assert want > 0
    assert sim.remove_dead_nodes() == want
    S.oracle_remove_dead(orc)
    for a in (A.ARR_NBR, A.ARR_VST, A.ARR_VINC, A.ARR_VLAST):
        assert np.array_equal(sim.get_array(a), orc.get_array(a)), A.ARRAY_NAMES[a]
    for chunk in (1, 9, 40, 50):
        sim.step(chunk)
        orc.step(chunk)
        assert sim.digest() == orc.digest(), f"digest differs at round {sim.round}"
        assert sim.counters().tolist() == orc.counters().tolist(), f"counters differ at round {sim.round}"
        assert sim.mismatches() == orc.mismatches()
    sim.close()
