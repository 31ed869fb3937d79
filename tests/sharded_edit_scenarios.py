"""Scenarios of the bulk membership calls (swim_sim_remove_dead_nodes, swim_sim_add_members) and of the push-pull
exchange (swim_sim_push_pull) on sharded handles, where they are collectives between steps. Shared by the emulator tests
(world 2 and 3, both exchanges) and the H100 tests (world 2 and 4 on one device). As in helpers.run_sharded, the ranks
are handles of one process, each driven by its own host thread, and the sum of the shards must be the single-shard
oracle's state: every local array concatenated over the ranks, the digest sum, the mismatch sum, the counter sums, and the
per-call totals summed over the ranks."""
import ctypes as C
import gc
import threading

import numpy as np
import pytest

from helpers import crash_events, default_config, generate_topology, random_events
from between_steps_oracle import push_pull as oracle_push_pull
from spec_fixture import msg
from swim_b200 import _abi as A
from view_edit_scenarios import dead_entries, oracle_add, oracle_remove_dead

NM = A.NO_MEMBER


class Shards:
    """`world` handles of one run, connected over peer memory ("p2p") or through NCCL ("nccl"; on the emulator the
    in-process stand-in of tests/emu/fake_nccl.cpp)."""

    def __init__(self, world, kw, nbr, mode="p2p", devices=None):
        from swim_b200.sim import Simulator
        self.sims = [Simulator(default_config(rank=r, world=world, device=(devices[r] if devices else -1), **kw))
                     for r in range(world)]
        for s in self.sims:
            s.set_view(nbr)
        if mode == "p2p":
            blobs = [s.ipc_export() for s in self.sims]
            for s in self.sims:
                s.ipc_connect(blobs)
        else:
            from swim_b200.sim import nccl_unique_id
            uid = nccl_unique_id()
            self.all(lambda s: s.connect(uid))

    def all(self, fn):
        """fn(sim) on every rank at once, one host thread each (a collective waits for its peers); the results in rank
        order. The first error is raised once every thread has finished.

        Python's cyclic garbage collector is run before the threads start and is off while they run. A handle left in a
        reference cycle by earlier code (a `pytest.raises` frame, say) is destroyed whenever the collector happens to
        run, in whichever thread allocates; swim_sim_destroy frees device memory, and cudaFree waits for every kernel on
        the device. Run in one rank's thread after its peers have launched their round kernels (which wait on the device
        for that rank) it would hold that rank back until the peers' watchdog fires. So no handle may be destroyed while
        the ranks of a run that share a device are stepping."""
        out, errs = [None] * len(self.sims), []

        def work(r):
            try:
                out[r] = fn(self.sims[r])
            except Exception as e:  # noqa: BLE001
                errs.append(e)
        ts = [threading.Thread(target=work, args=(r,)) for r in range(len(self.sims))]
        gc.collect()
        was_on = gc.isenabled()
        gc.disable()
        try:
            for t in ts:
                t.start()
            for t in ts:
                t.join()
        finally:
            if was_on:
                gc.enable()
        if errs:
            raise errs[0]
        return out

    def inject(self, events):
        for s in self.sims:
            s.inject(events)

    def step(self, rounds):
        self.all(lambda s: s.step(rounds))

    def total(self, fn):
        """Per-call totals summed over the ranks."""
        got = self.all(fn)
        return tuple(int(x) for x in np.sum(np.array(got, dtype=np.int64).reshape(len(got), -1), axis=0)) \
            if isinstance(got[0], tuple) else int(sum(got))

    def array(self, a):
        return self.sims[0].get_array(a) if a in A.REPLICATED_ARRAYS else np.concatenate([s.get_array(a) for s in self.sims])

    def check(self, ref, where):
        assert sum(s.digest() for s in self.sims) % 2 ** 64 == ref.digest() % 2 ** 64, f"{where}: digest differs"
        assert sum(s.mismatches() for s in self.sims) == ref.mismatches(), f"{where}: mismatch count differs"
        assert np.sum([s.counters() for s in self.sims], axis=0).tolist() == ref.counters().tolist(), f"{where}: counters"
        for a in range(A.ARR_COUNT):
            got, want = self.array(a), ref.get_array(a)
            if not np.array_equal(got, want):
                idx = np.flatnonzero(got != want)[:8]
                raise AssertionError(f"{where}: array {A.ARRAY_NAMES[a]} differs at {idx.tolist()}: "
                                     f"shards={got[idx].tolist()} reference={want[idx].tolist()}")

    def close(self):
        for s in self.sims:
            s.close()


def config(n, seed, **kw):
    base = dict(n_nodes=n, k_indirect=3, fanout=4, pb_cap=6, suspicion_rounds=3, retransmit=5, seed=seed)
    base.update(kw)
    return base


def setup(world, n, deg, mode, seed, devices=None, events=True, rounds=20, **kw):
    """Shards and the single-shard oracle on one random view, with the same event trace. `kw` overrides config fields;
    the view is generated at its view_cap (32 by default)."""
    from oracle.oracle import Oracle
    kw = config(n, seed, **kw)
    nbr = generate_topology("random", n, kw.get("view_cap", 32), deg, seed=seed)
    sh = Shards(world, kw, nbr, mode, devices)
    orc = Oracle(default_config(**kw))
    orc.set_view(nbr)
    if events:
        ev = random_events(np.random.default_rng(seed), n, rounds, n_crash=max(2, n // 12), n_rejoin=max(1, n // 40),
                           n_inject=n // 10)
        sh.inject(ev)
        orc.inject(ev)
    return sh, orc


def step(sh, orc, chunks):
    for c in chunks:
        sh.step(c)
        orc.step(c)
        sh.check(orc, f"round {orc.round}")


def push_pull(sh, orc, where):
    got, want = sh.total(lambda s: s.push_pull()), oracle_push_pull(orc)
    assert got == want, (where, got, want)
    sh.check(orc, f"after push_pull, {where}")
    return got


def remove_dead_then_rounds(world, n, mode, devices=None, chunks=(1, 1, 4, 10), **kw):
    """removeDeadNodes on every store of every rank, then rounds (the first one rebuilds the mail graph together)."""
    sh, orc = setup(world, n, 24, mode, seed=3, devices=devices, **{"loss_ppm": 20000, **kw})
    step(sh, orc, [6, 14])
    want = dead_entries(orc)
    assert want > 0
    assert sh.total(lambda s: s.remove_dead_nodes()) == want
    oracle_remove_dead(orc)
    sh.check(orc, "after remove_dead_nodes")
    step(sh, orc, chunks)
    sh.close()


def remove_dead_min_age(world, n, mode, min_age, devices=None, chunks=(1, 3, 8)):
    """min_age > 0 (which the oracle's call does not take): against the single-shard handle on the same inputs, whose
    own call is checked against a NumPy compaction of the oracle's rows in test_emu_view_edits.py."""
    from swim_b200.sim import Simulator
    kw = config(n, 4, suspicion_rounds=2)
    nbr = generate_topology("random", n, 32, 24, seed=4)
    sh = Shards(world, kw, nbr, mode, devices)
    one = Simulator(default_config(device=devices[0] if devices else -1, **kw))
    one.set_view(nbr)
    rng = np.random.default_rng(4)
    for r in (2, 6, 10, 14):  # Dead entries of several ages
        ev = crash_events(r, rng.choice(n, size=max(1, n // 25), replace=False))
        sh.inject(ev)
        one.inject(ev)
    sh.step(24)
    one.step(24)
    sh.check(one, "before")
    want = one.remove_dead_nodes(min_age)
    assert want > 0 and dead_entries(one) > 0, "the ages must straddle min_age"
    assert sh.total(lambda s: s.remove_dead_nodes(min_age)) == want
    sh.check(one, "after remove_dead_nodes")
    for c in chunks:
        sh.step(c)
        one.step(c)
        sh.check(one, f"round {one.round}")
    sh.close()
    one.close()


def add_members_then_rounds(world, n, mode, devices=None, chunks=(1, 2, 8), deg=26, **kw):
    """The same global add list on every rank; each applies the adds of its own observers. Adds to full rows, adds whose
    observer lies on another rank than the member, known members and duplicates within the call."""
    sh, orc = setup(world, n, deg, mode, seed=5, devices=devices, events=False, **{"loss_ppm": 10000, **kw})
    ev = crash_events(2, np.random.default_rng(5).choice(n, size=max(1, n // 30), replace=False))
    sh.inject(ev)
    orc.inject(ev)
    step(sh, orc, [6])
    rng = np.random.default_rng(5)
    k = max(40, n // 2)
    obs = rng.integers(0, n, size=k)
    obs[: k // 4] = obs[0]  # one observer gets many: its row fills up
    obs[k // 4: k // 2] = n - 1  # the last shard's last row (the smallest shard, when the split is uneven)
    mem = rng.integers(0, n, size=k)
    mem[obs == mem] = (mem[obs == mem] + 1) % n
    known = orc.get_array(A.ARR_NBR).reshape(n, -1)[obs[3 * k // 4:], 0]  # slot 0 of a row: a member it lists
    mem[3 * k // 4:] = np.where(known != NM, known, mem[3 * k // 4:])
    mem[-3:], obs[-3:] = mem[-4], obs[-4]  # duplicates within the call
    inc = rng.integers(0, 5, size=k)
    got = sh.total(lambda s: s.add_members(obs, mem, inc))
    want = oracle_add(orc, obs, mem, inc)
    assert got == want and want[0] > 0 and want[1] > 0, (got, want)
    per = sh.sims[0].cfg.n_nodes // world
    assert (obs // max(per, 1) != mem // max(per, 1)).any()
    sh.check(orc, "after add_members")
    step(sh, orc, chunks)
    sh.close()


def push_pull_inserts_then_rounds(world, n, mode, devices=None, rounds=50, chunk=10):
    """D < cap: push_pull inserts members on every rank; the next step rebuilds the mail graph, and 50 rounds after it
    stay equal to the oracle."""
    sh, orc = setup(world, n, 12, mode, seed=6, devices=devices, events=False, loss_ppm=10000)
    ev = crash_events(2, np.random.default_rng(6).choice(n, size=max(1, n // 25), replace=False))
    sh.inject(ev)
    orc.inject(ev)
    step(sh, orc, [4])
    got = push_pull(sh, orc, "inserts")
    assert got[0] > 0 and got[1] > 0, got
    step(sh, orc, [chunk] * (rounds // chunk))
    sh.close()


def push_pull_every(world, n, mode, rounds=24, every=6, devices=None, flags=0, churn=None, loss=20000, suspicion_max=0,
                    **overrides):
    """push_pull every `every` rounds under events, device churn and loss, in the protocol variants."""
    kw = dict(loss_ppm=loss, flags=flags, suspicion_max=suspicion_max, **overrides)
    if churn:
        kw.update(churn_ppm=churn[0], rejoin_min=churn[1], rejoin_max=churn[2])
    sh, orc = setup(world, n, 20, mode, seed=7, devices=devices, rounds=rounds, **kw)
    tot = np.zeros(3, dtype=np.int64)
    for _ in range(0, rounds, every):
        step(sh, orc, [every])
        tot += push_pull(sh, orc, f"round {orc.round}")
    step(sh, orc, [1, 2])
    assert tot[0] > 0 and tot[1] > 0, tot
    sh.close()


def edit_save_load(world, n, mode, devices=None):
    """An edit drops the checkpoint and refuses save until the next step; after that step save / load work on every
    rank, and a push_pull with inserts drops the checkpoint again."""
    from swim_b200._lib import SwimError
    sh, orc = setup(world, n, 16, mode, seed=8, devices=devices, rounds=12)
    step(sh, orc, [12])
    sh.all(lambda s: s.save())
    assert sh.total(lambda s: s.remove_dead_nodes()) == dead_entries(orc) > 0
    oracle_remove_dead(orc)
    for call in (lambda s: s.save(), lambda s: s.load()):
        for s in sh.sims:
            with pytest.raises(SwimError) as e:
                call(s)
            assert e.value.code == A.ESTATE
    step(sh, orc, [1])
    sh.all(lambda s: s.save())
    sh.step(5)
    sh.all(lambda s: s.load())
    sh.check(orc, "after load")
    step(sh, orc, [2, 3])
    assert push_pull(sh, orc, "inserts")[1] > 0
    for s in sh.sims:
        with pytest.raises(SwimError) as e:
            s.load()
        assert e.value.code == A.ESTATE
    step(sh, orc, [1, 4])
    sh.close()


def scalar_insert_refused(world, n, mode, devices=None):
    """A scalar insert on one rank is that rank's alone: its next step is refused (SWIM_ESTATE) before any collective,
    as before sharded bulk calls existed. A bulk call on the handle does not lift the refusal."""
    from swim_b200._lib import SwimError, lib
    sh, orc = setup(world, n, 10, mode, seed=9, devices=devices, events=False)
    step(sh, orc, [2])
    last = sh.sims[-1]
    first, count = C.c_uint32(), C.c_uint32()
    lib().swim_sim_local_range(last._h, C.byref(first), C.byref(count))
    node = first.value + count.value - 1
    listed = set(orc.get_array(A.ARR_NBR).reshape(n, 32)[node].tolist())
    member = next(m for m in range(n) if m != node and m not in listed)
    out, has = A.Message(), C.c_int()
    assert lib().swim_alive_node(last._h, node, C.byref(msg(A.MSG_ALIVE, member, 1)), C.byref(out), C.byref(has)) == 0
    for _ in range(2):
        with pytest.raises(SwimError) as e:
            last.step(1)
        assert e.value.code == A.ESTATE
    sh.close()


def not_connected_refused(n=40):
    """A sharded handle that is not connected to its peers refuses the three calls (SWIM_ESTATE) and changes nothing."""
    from swim_b200._lib import SwimError
    from swim_b200.sim import Simulator
    shard = Simulator(default_config(n_nodes=n, world=2, rank=1))
    shard.set_view(generate_topology("random", n, 32, 16, seed=12))
    before = shard.state()
    for call in (lambda: shard.remove_dead_nodes(), lambda: shard.add_members([30], [1]), lambda: shard.push_pull()):
        with pytest.raises(SwimError) as e:
            call()
        assert e.value.code == A.ESTATE
    after = shard.state()
    assert all(np.array_equal(before[k], after[k]) for k in before)
    shard.close()


def large_equals_single_shard(n, world, devices):
    """No rounds (every rank's round kernel would need the whole device): at n nodes, push_pull, remove_dead_nodes and
    add_members on the shards give the single-shard handle's arrays and totals. Suspect / Dead entries and incarnations
    are written into the rows first."""
    from swim_b200.sim import Simulator
    kw = config(n, 10, suspicion_rounds=4)
    nbr = generate_topology("random", n, 32, 16, seed=10)
    sh = Shards(world, kw, nbr, "p2p", devices)
    one = Simulator(default_config(device=devices[0], **kw))
    one.set_view(nbr)
    rng = np.random.default_rng(10)
    vst = one.get_array(A.ARR_VST)
    occ = vst != A.VACANT
    live = rng.choice([A.ALIVE, A.ALIVE, A.SUSPECT, A.DEAD], size=vst.shape).astype(np.uint8)
    vst = np.where(occ, live | np.where(live == A.SUSPECT, 2 << 2, 0).astype(np.uint8), A.VACANT).astype(np.uint8)
    vinc = np.where(occ, rng.integers(0, 4, size=vst.shape), 0).astype(np.uint32)
    alive = (rng.random(n) > 0.05).astype(np.uint8)
    per = (n + world - 1) // world
    for a, v in ((A.ARR_VST, vst), (A.ARR_VINC, vinc)):
        one.set_array(a, v)
        for r, s in enumerate(sh.sims):
            s.set_array(a, v[r * per * 32: min(n, (r + 1) * per) * 32])
    one.set_array(A.ARR_ALIVE, alive)
    for s in sh.sims:
        s.set_array(A.ARR_ALIVE, alive)

    def same(where):
        for a in range(A.ARR_COUNT):
            assert np.array_equal(sh.array(a), one.get_array(a)), (where, A.ARRAY_NAMES[a])
    want = one.push_pull()
    assert sh.total(lambda s: s.push_pull()) == want and want[1] > 0, want
    same("push_pull")
    want = one.remove_dead_nodes()
    assert sh.total(lambda s: s.remove_dead_nodes()) == want > 0
    same("remove_dead_nodes")
    obs = rng.integers(0, n, size=n // 4)
    mem = (obs + rng.integers(1, n, size=len(obs))) % n
    want = one.add_members(obs, mem, 2)
    assert sh.total(lambda s: s.add_members(obs, mem, 2)) == want and want[0] > 0
    same("add_members")
    want = one.push_pull()
    assert sh.total(lambda s: s.push_pull()) == want
    same("second push_pull")
    sh.close()
    one.close()


def tiny_last_shard(world, n, mode, devices=None):
    """Shards of very unequal size (n = 7 on 3 ranks: 3, 3 and 1 rows): every call and the rebuilds after them."""
    sh, orc = setup(world, n, 2, mode, seed=11, devices=devices, rounds=8)
    step(sh, orc, [3])
    assert push_pull(sh, orc, "inserts")[1] > 0
    step(sh, orc, [1, 4])
    obs, mem = [n - 1, n - 1, 0, 3], [0, 2, n - 1, 1]
    assert sh.total(lambda s: s.add_members(obs, mem, 1)) == oracle_add(orc, obs, mem, [1] * 4)
    sh.check(orc, "after add_members")
    step(sh, orc, [1, 5])
    assert sh.total(lambda s: s.remove_dead_nodes()) == dead_entries(orc)
    oracle_remove_dead(orc)
    step(sh, orc, [1, 6])
    push_pull(sh, orc, "last")
    step(sh, orc, [2])
    sh.close()
