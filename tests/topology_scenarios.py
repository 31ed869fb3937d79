"""Scenarios of the device view generator (swim_sim_generate_view), shared by the emulator tests (small sizes) and the
H100 tests (2^16 nodes and up): the generated matrix against the host generator's, the handle state against a
set_view of that matrix, sharded handles against one shard, and a run on symmetric views against the oracle."""
import numpy as np
import pytest

from helpers import assert_same_state, crash_events, default_config, generate_topology
from swim_b200 import _abi as A
from swim_b200._lib import SwimError
from swim_b200.sim import Simulator

# the arrays swim_sim_set_view writes, and every other array still at its initial value
VIEW_ARRAYS = (A.ARR_NBR, A.ARR_VST, A.ARR_VINC, A.ARR_VLAST)


def device_equals_host(kind, n, cap, deg, seed, full_state=True, steps=0):
    """generate_view's rows equal generate_topology's; with full_state the whole handle equals one given that matrix by
    set_view (state arrays and digest, then `steps` rounds of both)."""
    want = generate_topology(kind, n, cap, deg, seed=seed)
    cfg = default_config(n_nodes=n, view_cap=cap, seed=seed, suspicion_rounds=3)
    sim = Simulator(cfg)
    sim.generate_view(kind, deg, seed)
    got = sim.get_array(A.ARR_NBR).reshape(n, cap)
    if not np.array_equal(got, want):
        bad = np.flatnonzero((got != want).any(axis=1))[:4]
        raise AssertionError(f"{kind} n={n} cap={cap} degree={deg} seed={seed}: rows {bad.tolist()} differ: "
                             f"device {got[bad[0]].tolist()} host {want[bad[0]].tolist()}")
    if full_state:
        ref = Simulator(cfg)
        ref.set_view(want)
        for a in range(A.ARR_COUNT):
            assert np.array_equal(sim.get_array(a), ref.get_array(a)), A.ARRAY_NAMES[a]
        assert sim.digest() == ref.digest()
        if steps:
            ev = crash_events(2, np.arange(0, n, 37))
            for s in (sim, ref):
                s.inject(ev)
                s.step(steps)
            assert sim.digest() == ref.digest() and sim.counters().tolist() == ref.counters().tolist()
            assert sim.mismatches() == ref.mismatches()
        ref.close()
    sim.close()


def sharded_equals_single(world, kind, n, deg, seed, devices=None):
    """Every rank generates the global matrix and keeps its rows: the ranks' arrays, concatenated, are the single shard's."""
    one = Simulator(default_config(n_nodes=n, seed=seed))
    one.generate_view(kind, deg, seed)
    ranks = [Simulator(default_config(n_nodes=n, seed=seed, rank=r, world=world, device=devices[r] if devices else -1))
             for r in range(world)]
    for s in ranks:
        s.generate_view(kind, deg, seed)
    for a in VIEW_ARRAYS + (A.ARR_ALIVE, A.ARR_SELF_INC):
        got = ranks[0].get_array(a) if a in A.REPLICATED_ARRAYS else np.concatenate([s.get_array(a) for s in ranks])
        assert np.array_equal(got, one.get_array(a)), A.ARRAY_NAMES[a]
    assert sum(s.digest() for s in ranks) % 2 ** 64 == one.digest()
    # as set_view: refused once the peers have mapped this rank's arrays
    blobs = [s.ipc_export() for s in ranks]
    for s in ranks:
        s.ipc_connect(blobs)
    with pytest.raises(SwimError) as e:
        ranks[0].generate_view(kind, deg, seed)
    assert e.value.code == A.ESTATE
    for s in ranks:
        s.close()
    one.close()


def symmetric_run_equals_oracle(n, deg, rounds, chunks, crashes, churn=None, loss=0, seed=5, crash_round=10):
    """A run on device-generated symmetric views equals the oracle fed the host matrix: digest, counters and convergence
    count after every chunk, every state array at the end."""
    from oracle.oracle import Oracle
    kw = dict(n_nodes=n, seed=seed, loss_ppm=loss)
    if churn:
        kw.update(churn_ppm=churn[0], rejoin_min=churn[1], rejoin_max=churn[2])
    cfg = default_config(**kw)
    sim = Simulator(cfg)
    sim.generate_view("symmetric", deg, seed)
    orc = Oracle(cfg)
    orc.set_view(generate_topology("symmetric", n, 32, deg, seed=seed))
    rng = np.random.default_rng(seed)
    ev = crash_events(crash_round, np.sort(rng.choice(n, size=crashes, replace=False)))
    sim.inject(ev)
    orc.inject(ev)
    assert sum(chunks) == rounds
    for c in chunks:
        sim.step(c)
        orc.step(c)
        assert sim.digest() == orc.digest(), f"digest differs at round {sim.round}"
        assert sim.counters().tolist() == orc.counters().tolist(), f"counters differ at round {sim.round}"
        assert sim.mismatches() == orc.mismatches(), f"convergence count differs at round {sim.round}"
    assert_same_state(sim, orc, f"round {sim.round}")
    sim.close()


def errors_and_checkpoint(n):
    """generate_view refuses what the host generator refuses, with the same code, and a new view drops the checkpoint."""
    sim = Simulator(default_config(n_nodes=n))
    for kind, deg in (("symmetric", 7), ("symmetric", 34), ("random", 33), ("ring", 40), (9, 8)):
        with pytest.raises(SwimError) as host:
            generate_topology(kind, n, 32, deg, seed=1)
        with pytest.raises(SwimError) as dev:
            sim.generate_view(kind, deg, 1)
        assert dev.value.code == host.value.code, (kind, deg)
    with pytest.raises(SwimError) as e:
        sim.step(1)
    assert e.value.code == A.ESTATE  # nothing was installed
    sim.generate_view("symmetric", 8, 3)
    sim.step(2)
    sim.save()
    sim.generate_view("ring", 8, 3)
    with pytest.raises(SwimError) as e:
        sim.load()
    assert e.value.code == A.ESTATE
    sim.close()
