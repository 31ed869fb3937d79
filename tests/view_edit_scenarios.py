"""Scenarios of the bulk membership edits (swim_sim_remove_dead_nodes, swim_sim_add_members) and of the device-built mail
graph (swim_sim_set_view_device), shared by the emulator tests (small sizes) and the H100 tests (2^16 nodes and up).
Every scenario is checked against the CPU oracle, whose membership calls act on one store at a time."""
import numpy as np
import pytest

from helpers import assert_same_state, crash_events, default_config, generate_topology, make_pair, random_events
from spec_fixture import msg
from swim_b200 import _abi as A
from swim_b200.sim import Simulator

NM = A.NO_MEMBER
SET_VIEW = Simulator.set_view  # (the sharded tests route Simulator.set_view through set_view_device below)


def emulated():
    import swim_b200._lib as L
    return L.SO_PATH.endswith("libswim_emu.so")


def with_hub(nbr, hub):
    """Every other row lists `hub` (a full row gives up its largest member for it)."""
    out = nbr.copy()
    rows = ~(out == hub).any(axis=1)
    rows[hub] = False
    out[rows, -1] = hub
    out.sort(axis=1)
    return out


def set_view_device(sim, nbr, dtype="uint32"):
    """swim_sim_set_view_device. On the emulator device memory is host memory, so a NumPy array's address is passed; on a
    GPU the matrix goes up as a torch tensor of `dtype` and Simulator.set_view hands its device pointer over."""
    nbr = np.ascontiguousarray(nbr, dtype=np.uint32)
    if emulated():
        from swim_b200._lib import check, lib
        check(lib().swim_sim_set_view_device(sim._h, nbr.ctypes.data), "swim_sim_set_view_device", sim._h)
        return
    import torch
    t = torch.from_numpy(nbr.view(np.int32)).cuda()
    SET_VIEW(sim, t if dtype == "int32" else t.view(torch.uint32))


def topology(kind, n, cap, deg, seed):
    if kind == "empty":
        return np.full((n, cap), NM, dtype=np.uint32)
    return generate_topology(kind, n, cap, deg, seed=seed)


def set_view_device_equals_set_view(n, cap, kind, deg, rounds, hub=None, vacant_rows=0, seed=1, dtype="uint32"):
    from swim_b200.sim import Simulator
    rng = np.random.default_rng(seed)
    cfg = default_config(n_nodes=n, view_cap=cap, seed=seed, loss_ppm=20000, suspicion_rounds=3)
    nbr = topology(kind, n, cap, deg, seed)
    if hub is not None:
        nbr = with_hub(nbr, hub)
    if vacant_rows:
        nbr[rng.choice(n, size=vacant_rows, replace=False)] = NM
    host, dev = make_pair(cfg, nbr)  # (host upload, oracle)
    sim = Simulator(cfg)
    set_view_device(sim, nbr, dtype)
    orc = dev
    ev = crash_events(2, rng.choice(n, size=max(1, n // 20), replace=False)) if n > 1 else crash_events(2, [0])
    for s in (sim, host, orc):
        s.inject(ev)
    assert_same_state(sim, orc, "after set_view_device")
    for r in range(rounds):
        for s in (sim, host, orc):
            s.step(1)
        assert_same_state(sim, orc, f"{kind} n={n} cap={cap} round {r + 1}")
        assert host.digest() == sim.digest()
    return sim, orc


def oracle_remove_dead(orc):
    for node in range(orc.first, orc.first + orc.n_local):
        orc.remove_dead_nodes(node)


def dead_entries(orc):
    return int(np.count_nonzero(orc.get_array(A.ARR_VST) & 3 == A.DEAD))


def remove_dead_then_step(n, deg, before, after, flags=0, loss=0, churn=None, every_round=True, seed=3):
    """Crashes, rounds until Dead entries exist, removeDeadNodes on every store, then more rounds: equal to the oracle."""
    rng = np.random.default_rng(seed)
    kw = dict(n_nodes=n, seed=seed, loss_ppm=loss, suspicion_rounds=3, flags=flags)
    if churn:
        kw.update(churn_ppm=churn[0], rejoin_min=churn[1], rejoin_max=churn[2])
    sim, orc = make_pair(default_config(**kw), generate_topology("random", n, 32, deg, seed=seed))
    ev = random_events(rng, n, before, n_crash=max(2, n // 10), n_rejoin=max(1, n // 40), n_inject=n // 10)
    sim.inject(ev)
    orc.inject(ev)
    sim.step(before)
    orc.step(before)
    want = dead_entries(orc)
    assert want > 0
    assert sim.remove_dead_nodes() == want
    oracle_remove_dead(orc)
    assert dead_entries(orc) == 0
    assert_same_state(sim, orc, "after remove_dead_nodes")
    chunks = [1] * after if every_round else [1, 4, after - 5]
    for c in chunks:
        sim.step(c)
        orc.step(c)
        assert_same_state(sim, orc, f"round {sim.round}")
    return sim, orc


def remove_dead_min_age(n, min_age, seed=4):
    """min_age > 0 against a NumPy compaction of the oracle's rows."""
    rng = np.random.default_rng(seed)
    sim, orc = make_pair(default_config(n_nodes=n, seed=seed, suspicion_rounds=2), generate_topology("random", n, 32, 24, seed=seed))
    for r in (2, 6, 10, 14):  # Dead entries of several ages
        ev = crash_events(r, rng.choice(n, size=max(1, n // 25), replace=False))
        sim.inject(ev)
        orc.inject(ev)
    sim.step(24)
    orc.step(24)
    cap = 32
    nb, st, inc, last = (orc.get_array(a).reshape(-1, cap) for a in (A.ARR_NBR, A.ARR_VST, A.ARR_VINC, A.ARR_VLAST))
    live = st & 3
    drop = (live == A.DEAD) & (np.uint32(orc.round) - last >= min_age)
    keep = (live != A.VACANT) & ~drop
    assert drop.any() and ((live == A.DEAD) & ~drop).any(), "the ages must straddle min_age"
    order = np.argsort(~keep, axis=1, kind="stable")
    kept = np.arange(cap)[None, :] < keep.sum(axis=1)[:, None]
    want = {a: np.where(kept, np.take_along_axis(x, order, 1), fill)
            for a, x, fill in ((A.ARR_NBR, nb, NM), (A.ARR_VST, st, A.VACANT), (A.ARR_VINC, inc, 0), (A.ARR_VLAST, last, 0))}
    assert sim.remove_dead_nodes(min_age) == int(drop.sum())
    for a, w in want.items():
        assert np.array_equal(sim.get_array(a), w.reshape(-1).astype(A.ARRAY_DTYPES[a])), A.ARRAY_NAMES[a]


def oracle_add(orc, observers, members, incs):
    from oracle.oracle import OracleError
    added = full = 0
    for o, m, i in zip(observers, members, incs):
        if int(m) in {x.id for x in orc.get_members(int(o))}:
            continue
        try:
            orc.alive_node(int(o), msg(A.MSG_ALIVE, int(m), int(i)))
            added += 1
        except OracleError as e:
            assert e.code == A.ECAP
            full += 1
    return added, full


def export_matches_oracle(sim, orc):
    from swim_b200.types import Alive, Dead, Suspect, decode

    def tup(m):
        kind = A.MSG_SUSPECT if isinstance(m, Suspect) else A.MSG_DEAD if isinstance(m, Dead) else A.MSG_ALIVE
        assert isinstance(m, (Suspect, Dead, Alive))
        return kind, int(m.node[1:]), m.incarnation, int(m.deadFrom[1:]) if kind == A.MSG_DEAD else 0
    got = sorted((s, d, tuple(tup(m) for m in decode(b).unEnvelope)) for s, d, b in sim.export_round())
    want = sorted((s, d, tuple((int(r["kind"]), int(r["member"]), int(r["incarnation"]), int(r["from"]) if r["kind"] == A.MSG_DEAD else 0)
                               for r in recs)) for s, d, recs in orc.sent())
    assert got == want
    return len(got)


def add_members_then_step(n, deg, n_adds, after, seed=5, every_round=True):
    """Unknown members inserted (Alive, given incarnation, lastChange = now), known ones and in-call duplicates left alone,
    adds to full rows dropped; then rounds equal to the oracle, and the next round's export equals its envelopes."""
    from swim_b200._lib import SwimError
    rng = np.random.default_rng(seed)
    sim, orc = make_pair(default_config(n_nodes=n, seed=seed, suspicion_rounds=3, loss_ppm=10000),
                         generate_topology("random", n, 32, deg, seed=seed))
    ev = crash_events(2, rng.choice(n, size=max(1, n // 30), replace=False))
    sim.inject(ev)
    orc.inject(ev)
    sim.step(6)
    orc.step(6)
    obs = rng.integers(0, n, size=n_adds)
    obs[: n_adds // 4] = obs[0]  # one observer gets many: its row fills up
    mem = rng.integers(0, n, size=n_adds)
    mem[obs == mem] = (mem[obs == mem] + 1) % n
    known = orc.get_array(A.ARR_NBR).reshape(n, 32)[obs[n_adds // 2:], 0]  # slot 0 of a row: a member it lists
    mem[n_adds // 2:] = np.where(known != NM, known, mem[n_adds // 2:])
    mem[-3:], obs[-3:] = mem[-4], obs[-4]  # duplicates within the call
    inc = rng.integers(0, 5, size=n_adds)
    before = sim.get_array(A.ARR_VINC)
    got = sim.add_members(obs, mem, inc)
    want = oracle_add(orc, obs, mem, inc)
    assert got == want and want[0] > 0 and want[1] > 0, (got, want)
    assert_same_state(sim, orc, "after add_members")
    assert not np.array_equal(before, sim.get_array(A.ARR_VINC)) or inc.max() == 0
    with pytest.raises(SwimError) as e:
        sim.export_round()
    assert e.value.code == A.ESTATE
    chunks = [1] * after if every_round else [1, after - 1]
    for c in chunks:
        sim.step(c)
        orc.step(c)
        assert_same_state(sim, orc, f"round {sim.round}")
        if c == 1:
            export_matches_oracle(sim, orc)
    return sim, orc


def error_paths(n):
    """EINVAL changes nothing; edits are single-shard only; an edit drops the checkpoint until the next save."""
    from swim_b200._lib import SwimError
    from swim_b200.sim import Simulator
    nbr = generate_topology("random", n, 32, 16, seed=9)
    sim, orc = make_pair(default_config(n_nodes=n, seed=9), nbr)
    ev = crash_events(2, [1, 2, 3])
    sim.inject(ev)
    orc.inject(ev)
    sim.step(12)
    orc.step(12)
    before = sim.state()
    for obs, mem in (([0], [n]), ([n], [0]), ([4, 5], [7, 5])):
        with pytest.raises(SwimError) as e:
            sim.add_members(obs, mem)
        assert e.value.code == A.EINVAL
    after = sim.state()
    assert all(np.array_equal(before[k], after[k]) for k in before)
    assert sim.add_members([], []) == (0, 0)
    assert_same_state(sim, orc, "after rejected adds")
    shard = Simulator(default_config(n_nodes=n, world=2, rank=0))
    shard.set_view(nbr)
    for call in (lambda: shard.remove_dead_nodes(), lambda: shard.add_members([0], [1])):
        with pytest.raises(SwimError) as e:
            call()
        assert e.value.code == A.ESTATE
    shard.close()
    sim.save()
    assert sim.remove_dead_nodes() > 0
    oracle_remove_dead(orc)
    for _ in range(2):  # before and after the step that rebuilds the mail graph
        with pytest.raises(SwimError) as e:
            sim.load()
        assert e.value.code == A.ESTATE
        sim.step(1)
        orc.step(1)
    sim.save()
    sim.step(3)
    sim.load()
    assert_same_state(sim, orc, "after load")
