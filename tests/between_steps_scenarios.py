"""What the scenarios of the calls between steps share: push_pull (DESIGN.md 2.6), join (2.7) and leave (2.8), each
named by its Simulator method. A call on a handle pair is checked against the CPU oracle's statement
(tests/between_steps_oracle.c): the outputs, every state array, the counters and the digest. The sharded scenarios run
on sharded_edit_scenarios' Shards and hold the shards' sums to the single-shard oracle."""
import numpy as np
import pytest

import sharded_edit_scenarios as SE
from between_steps_oracle import join as oracle_join, leave as oracle_leave, push_pull as oracle_push_pull
from helpers import assert_same_state, default_config, generate_topology, make_pair
from swim_b200 import _abi as A

ORACLE = {"push_pull": oracle_push_pull, "join": oracle_join, "leave": oracle_leave}


def call(name, sim, orc, *args, where="", **kw):
    """One call on the handle and on the oracle: the same outputs and the same state after it."""
    got, want = getattr(sim, name)(*args, **kw), ORACLE[name](orc, *args, **kw)
    assert got == want, (where, got, want)
    assert_same_state(sim, orc, f"after {name}, {where}")
    return got


def step(sim, orc, rounds, check=True):
    sim.step(rounds)
    orc.step(rounds)
    if check:
        assert_same_state(sim, orc, f"round {sim.round}")


def pair(n, cap=32, deg=32, kind="random", seed=1, nbr=None, **kw):
    kw.setdefault("suspicion_rounds", 3)
    cfg = default_config(n_nodes=n, view_cap=cap, seed=seed, **kw)
    return make_pair(cfg, generate_topology(kind, n, cap, deg, seed=seed) if nbr is None else nbr)


def same_state(before, after):
    return all(np.array_equal(before[k], after[k]) for k in before)


def error_paths(name, args, invalid=(), n=40):
    """SWIM_EINVAL on each argument list of `invalid`, before anything changes; SWIM_ESTATE with `args` on a sharded
    handle that is not connected and before a view is installed."""
    from swim_b200._lib import SwimError
    from swim_b200.sim import Simulator
    if invalid:
        sim, orc = pair(n, 32, 10, seed=11)
        before = sim.state()
        for bad in invalid:
            with pytest.raises(SwimError) as e:
                getattr(sim, name)(*bad)
            assert e.value.code == A.EINVAL
        assert same_state(before, sim.state())
        sim.close()
    shard = Simulator(default_config(n_nodes=n, world=2, rank=0))
    shard.set_view(generate_topology("random", n, 32, 16, seed=12))
    bare = Simulator(default_config(n_nodes=n))
    for s in (shard, bare):
        with pytest.raises(SwimError) as e:
            getattr(s, name)(*args)
        assert e.value.code == A.ESTATE
        s.close()


# ------------------------------------------------------------------ sharded handles
def sharded_every(name, args, world, n, mode, devices=None, rounds=24, every=6, **kw):
    """The call with args(k) every `every` rounds on `world` ranks, under events and loss; the shards' sums against the
    single-shard oracle after every call and every chunk. The first two outputs, summed, are positive. `kw` overrides
    config fields (the view is generated at its view_cap)."""
    sh, orc = SE.setup(world, n, 14, mode, seed=13, devices=devices, rounds=rounds, **{"loss_ppm": 10000, **kw})
    tot = 0
    for k in range(rounds // every):
        SE.step(sh, orc, [every])
        a = args(k)
        got, want = sh.total(lambda s: getattr(s, name)(*a)), ORACLE[name](orc, *a)
        assert got == want, (k, got, want)
        sh.check(orc, f"after {name} {k}")
        tot = tot + np.array(got, dtype=np.int64)
    SE.step(sh, orc, [1, 3])
    assert tot[0] > 0 and tot[1] > 0, tot
    sh.close()


def sharded_equals_single_shard(name, args, n, world, devices, mode="p2p", **kw):
    """No rounds: at n nodes, with 5 % of them down, two calls with args(rng, k) on the shards and on the single-shard
    handle give the same arrays and totals, and the second output is positive. `kw` overrides config fields."""
    from swim_b200.sim import Simulator
    kw = SE.config(n, 14, **{"suspicion_rounds": 4, **kw})
    nbr = generate_topology("random", n, kw.get("view_cap", 32), 16, seed=14)
    sh = SE.Shards(world, kw, nbr, mode, devices)
    one = Simulator(default_config(device=devices[0] if devices else -1, **kw))
    one.set_view(nbr)
    rng = np.random.default_rng(14)
    alive = (rng.random(n) > 0.05).astype(np.uint8)
    one.set_array(A.ARR_ALIVE, alive)
    for s in sh.sims:
        s.set_array(A.ARR_ALIVE, alive)
    for k in range(2):
        a = args(rng, k)
        want = getattr(one, name)(*a)
        assert sh.total(lambda s: getattr(s, name)(*a)) == want and want[1] > 0, want
        for x in range(A.ARR_COUNT):
            assert np.array_equal(sh.array(x), one.get_array(x)), (k, A.ARRAY_NAMES[x])
    sh.close()
    one.close()


def sharded_not_connected(name, args, n=40):
    """SWIM_ESTATE on a sharded handle that is not connected, and nothing changes."""
    from swim_b200._lib import SwimError
    from swim_b200.sim import Simulator
    shard = Simulator(default_config(n_nodes=n, world=2, rank=1))
    shard.set_view(generate_topology("random", n, 32, 16, seed=12))
    before = shard.state()
    with pytest.raises(SwimError) as e:
        getattr(shard, name)(*args)
    assert e.value.code == A.ESTATE
    assert same_state(before, shard.state())
    shard.close()
