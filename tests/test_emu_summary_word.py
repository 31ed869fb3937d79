"""The scans decide from a 4-byte summary word per node (SimDev::nsum: process up, piggyback count, min(L, 4), a Suspect
slot, exposed) and gather the meta bitmaps only for exposed nodes. These cases, on the emulator against the oracle, aim at
the writers of that word and at the decisions that skip the bitmaps: crashes that expose a row while an INJECT rewrites it,
crash / rejoin / crash of one member, loss without bitmaps for every P and round-robin order, wide rows, parameter changes,
checkpoints in the middle of a burst, membership edits and sharded runs."""
import numpy as np
import pytest

import view_edit_scenarios as S
from helpers import assert_same_state, concat_events, default_config, generate_topology, make_pair, run_sharded
from swim_b200 import _abi as A
from swim_b200.sim import make_events
from emu_fixtures import emu_library  # noqa: F401  (autouse fixtures)


def _inject(sim, orc, ev):
    sim.inject(ev)
    orc.inject(ev)


def _steps(sim, orc, chunks, what):
    for c in chunks:
        sim.step(c)
        orc.step(c)
        assert_same_state(sim, orc, f"{what}, round {sim.round}")


def _row_crash_with_inject(n=96, seed=1):
    """Several members of one row crash in the same round as INJECTs on that row (Alive about a crashed member with a new
    incarnation, Suspect about another member); later the same on a row whose entries are already Suspect or Dead."""
    cfg = default_config(n_nodes=n, seed=seed, suspicion_rounds=4, k_indirect=3, fanout=3)
    nbr = generate_topology("random", n, 32, 24, seed=seed)
    sim, orc = make_pair(cfg, nbr)
    rows = nbr.reshape(n, 32)
    evs = []
    for r, obs in ((3, 10), (9, 10), (9, 41)):
        members = [int(m) for m in rows[obs][:24:5]]
        evs.append(make_events(np.full(len(members), r, np.uint32), np.array(members, np.uint32),
                               np.full(len(members), A.EV_CRASH, np.uint8)))
        evs.append(make_events(np.array([r, r], np.uint32), np.array([obs, obs], np.uint32),
                               np.full(2, A.EV_INJECT, np.uint8),
                               msg_kind=np.array([A.MSG_ALIVE, A.MSG_SUSPECT], np.uint8),
                               msg_node=np.array([members[0], int(rows[obs][1])], np.uint32),
                               msg_inc=np.array([7, 3]), msg_from=np.array([0, 0], np.uint32)))
    _inject(sim, orc, concat_events(evs))
    return sim, orc


@pytest.mark.parametrize("xmode", ["1", "0"])
def test_row_crash_burst_with_inject(xmode, monkeypatch):
    monkeypatch.setenv("SWIM_XMODE", xmode)
    sim, orc = _row_crash_with_inject()
    _steps(sim, orc, [1] * 14 + [40], f"xmode {xmode}")


@pytest.mark.parametrize("chunks", [[1] * 24, [2, 40]])
def test_crash_rejoin_crash_of_one_member(chunks):
    n = 80
    cfg = default_config(n_nodes=n, seed=12, suspicion_rounds=3)
    nbr = generate_topology("random", n, 32, 20, seed=4)
    sim, orc = make_pair(cfg, nbr)
    m = 17
    ev = make_events(np.array([2, 6, 9, 15], np.uint32), np.full(4, m, np.uint32),
                     np.array([A.EV_CRASH, A.EV_REJOIN, A.EV_CRASH, A.EV_REJOIN], np.uint8))
    _inject(sim, orc, ev)
    _steps(sim, orc, chunks, "crash / rejoin / crash")


@pytest.mark.parametrize("flags", [0, A.F_ROUND_ROBIN])
@pytest.mark.parametrize("probes", [1, 2, 3, 4])
def test_loss_without_bitmaps(probes, flags):
    """Under loss every live node depends on its draws; nodes that are not exposed decide from their loss draws alone."""
    n = 200
    cfg = default_config(n_nodes=n, seed=30 + probes, probes_per_round=probes, loss_ppm=150000, suspicion_rounds=3,
                         flags=flags)
    nbr = generate_topology("random", n, 32, 14, seed=probes)
    sim, orc = make_pair(cfg, nbr)
    rng = np.random.default_rng(probes)
    _inject(sim, orc, make_events(np.full(8, 4, np.uint32), rng.choice(n, 8, replace=False).astype(np.uint32),
                                  np.full(8, A.EV_CRASH, np.uint8)))
    _steps(sim, orc, [1] * 6 + [5, 33], f"P {probes} flags {flags}")


@pytest.mark.parametrize("cap", [64, 128, 256])
@pytest.mark.parametrize("loss", [0, 40000])
def test_wide_rows(cap, loss):
    n = 150
    cfg = default_config(n_nodes=n, view_cap=cap, seed=cap + loss, loss_ppm=loss, suspicion_rounds=4, probes_per_round=2)
    nbr = generate_topology("random", n, cap, min(cap - 5, n - 1), seed=7)
    sim, orc = make_pair(cfg, nbr)
    rng = np.random.default_rng(cap)
    crashed = rng.choice(n, 14, replace=False).astype(np.uint32)
    ev = concat_events([make_events(np.full(14, 3, np.uint32), crashed, np.full(14, A.EV_CRASH, np.uint8)),
                        make_events(np.full(4, 8, np.uint32), crashed[:4], np.full(4, A.EV_REJOIN, np.uint8))])
    _inject(sim, orc, ev)
    _steps(sim, orc, [1] * 10 + [36], f"cap {cap} loss {loss}")


def test_set_params_mid_run():
    """Loss and round-robin order switched on and off between steps: the scans change how they decide (staged picks, loss
    draws) on summary words written under the old parameters. Each stretch is compared with a fresh oracle of the new
    parameters that starts from the state the stretch started from."""
    from oracle.oracle import Oracle
    n = 160
    kw = dict(n_nodes=n, seed=5, suspicion_rounds=5, probes_per_round=3)
    nbr = generate_topology("random", n, 32, 16, seed=9)
    sim, orc = make_pair(default_config(**kw), nbr)
    rng = np.random.default_rng(5)
    _inject(sim, orc, make_events(np.full(12, 2, np.uint32), rng.choice(n, 12, replace=False).astype(np.uint32),
                                  np.full(12, A.EV_CRASH, np.uint8)))
    _steps(sim, orc, [1, 1, 2], "before set_params")
    for params in (dict(loss_ppm=100000), dict(loss_ppm=100000, flags=A.F_ROUND_ROBIN), dict(loss_ppm=0, flags=0)):
        sim.set_params(**params)
        kw.update(params)
        nxt = Oracle(default_config(**kw))
        nxt.set_view(nbr)
        for a in range(A.ARR_COUNT):
            if a != A.ARR_NBR:  # (the view itself is the same)
                nxt.set_array(a, orc.get_array(a))
        nxt.set_round(orc.round)
        orc, c0 = nxt, sim.counters()
        for c in (1, 1, 3, 12):
            sim.step(c)
            orc.step(c)
            for a in range(A.ARR_COUNT):
                assert np.array_equal(sim.get_array(a), orc.get_array(a)), (params, sim.round, A.ARRAY_NAMES[a])
            assert (sim.counters() - c0).tolist() == orc.counters().tolist(), (params, sim.round)
            assert sim.digest() == orc.digest() and sim.mismatches() == orc.mismatches(), (params, sim.round)


@pytest.mark.parametrize("xmode", ["1", "0"])
def test_save_load_mid_burst(xmode, monkeypatch):
    """A checkpoint taken in the middle of a crash burst (exposed rows, some with spurious exposed bits after a rejoin)
    and replayed twice."""
    monkeypatch.setenv("SWIM_XMODE", xmode)
    sim, orc = _row_crash_with_inject(seed=2)
    rng = np.random.default_rng(2)
    crashed = rng.choice(96, 10, replace=False).astype(np.uint32)
    _inject(sim, orc, concat_events([make_events(np.full(10, 4, np.uint32), crashed, np.full(10, A.EV_CRASH, np.uint8)),
                                     make_events(np.full(5, 6, np.uint32), crashed[:5], np.full(5, A.EV_REJOIN, np.uint8))]))
    _steps(sim, orc, [1] * 7, "burst")
    sim.save()
    _steps(sim, orc, [1, 2, 40], "after save")
    ref = (sim.digest(), sim.counters().tolist(), sim.mismatches())
    for _ in range(2):
        sim.load()
        sim.step(1)
        sim.step(2)
        sim.step(40)
        assert (sim.digest(), sim.counters().tolist(), sim.mismatches()) == ref


def test_remove_dead_nodes_then_steps():
    S.remove_dead_then_step(n=180, deg=24, before=14, after=6, every_round=False, churn=(20000, 2, 6))


def test_add_members_then_steps():
    S.add_members_then_step(n=150, deg=20, n_adds=60, after=6, every_round=False)


@pytest.mark.parametrize("world", [2, 3])
def test_sharded(world, monkeypatch):
    """Shards whose first node is not a multiple of four (n = 301: the scans' unaligned path) and aligned ones."""
    monkeypatch.setenv("SWIM_XMODE", "1")
    run_sharded(world, n=301, chunks=[1, 1, 3, 36], loss=0, deg=24)
    run_sharded(world, n=400, chunks=[2, 30], loss=20000, deg=20)
