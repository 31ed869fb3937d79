"""Scenarios of the seed joins between steps (swim_sim_join, DESIGN.md 2.7), shared by the emulator tests (small sizes)
and the H100 tests (2^16 nodes and up). Every call is checked against the CPU oracle's statement
(tests/between_steps_oracle.c, oracle_join): the three outputs, every state array, the counters and the digest. The
sharded scenarios hold the shards' sums to the single-shard oracle (between_steps_scenarios)."""
from functools import partial

import numpy as np
import pytest

import between_steps_scenarios as B
from between_steps_oracle import join as oracle_join, push_pull as oracle_push_pull
from between_steps_scenarios import pair, step
from helpers import assert_same_state, crash_events, random_events
from swim_b200 import _abi as A

join = partial(B.call, "join")


def restart_pairs(rng, n, hosts, frac=0.05):
    """A share of the nodes each joining through every one of `hosts` (a node never joins through itself)."""
    who = rng.choice(n, size=max(2, int(n * frac)), replace=False)
    nodes = np.repeat(who, len(hosts))
    seeds = np.tile(hosts, len(who))
    keep = nodes != seeds
    return nodes[keep], seeds[keep]


def join_every(n, cap, deg, rounds=24, every=6, seed=1, hosts=3, **kw):
    """Steps with events (crashes, rejoins, injected records), churn and loss as given, and every `every` rounds a join
    of 5 % of the nodes through `hosts` fixed seeds, alternately fresh and not. Returns the summed outputs."""
    sim, orc = pair(n, cap, deg, seed=seed, **kw)
    rng = np.random.default_rng(seed)
    ev = random_events(rng, n, rounds, n_crash=max(2, n // 12), n_rejoin=max(1, n // 30), n_inject=max(1, n // 8))
    sim.inject(ev)
    orc.inject(ev)
    seeds = rng.choice(n, size=hosts, replace=False)
    tot = np.zeros(3, dtype=np.int64)
    for k, _ in enumerate(range(0, rounds, every)):
        step(sim, orc, every, check=False)
        nodes, sd = restart_pairs(rng, n, seeds)
        tot += join(sim, orc, nodes, sd, fresh=k % 2 == 1, where=f"n={n} cap={cap} round {sim.round}")
    step(sim, orc, 2)
    return sim, orc, tot


def edge_cases(n=120):
    """Empty joiner rows, a joiner that does not list its seed, mutual and duplicated pairs, a hub seed, a down seed and
    a down joiner, and n = 0."""
    sim, orc = pair(n, 32, 6, "ring", seed=2)
    crashed = [5, 40]
    ev = crash_events(1, crashed)
    sim.inject(ev)
    orc.inject(ev)
    step(sim, orc, 3)
    assert sim.join([], []) == (0, 0, 0)
    assert_same_state(sim, orc, "n = 0")
    nbr = orc.get_array(A.ARR_NBR).reshape(n, 32)
    assert 60 not in nbr[10] and 10 not in nbr[60]
    got = join(sim, orc, [10], [60], where="neither lists the other")
    assert got[0] == 1 and got[1] > 0
    join(sim, orc, [70, 70, 80, 90], [71, 71, 90, 80], where="duplicated and mutual pairs")
    got = join(sim, orc, [5, 41, 42], [43, 40, 45], where="a down joiner, a down seed")
    assert got[0] == 1, got
    got = join(sim, orc, [20, 21, 22], [100, 101, 102], fresh=True, where="fresh joiners")
    assert got[0] == 3 and got[1] > 0, got
    join(sim, orc, [5, 30], [31, 5], fresh=True, where="a down fresh joiner is left alone")
    hub = n // 2
    others = np.array([i for i in range(n) if i != hub])
    join(sim, orc, others, np.full(len(others), hub), where="a hub seed")
    step(sim, orc, 4)
    # empty rows on both sides: two fresh joiners that name each other send Alive(self) only
    sim2, orc2 = pair(40, 32, 8, seed=3)
    got = join(sim2, orc2, [1, 2], [2, 1], fresh=True, where="two empty rows")
    assert got == (2, 2, 0), got
    step(sim2, orc2, 3)


def hub(n, joiners, cap=32, deg=8, seed=4, fresh=True):
    """Thousands of joiners through one seed: the seed's row fills (inserts dropped), every joiner learns the seed's
    members; then rounds."""
    sim, orc = pair(n, cap, deg, seed=seed, loss_ppm=10000)
    step(sim, orc, 2)
    rng = np.random.default_rng(seed)
    h = int(rng.integers(0, n))
    who = rng.choice(np.delete(np.arange(n), h), size=joiners, replace=False)
    got = join(sim, orc, who, np.full(joiners, h), fresh=fresh, where="hub")
    assert got[0] == joiners and got[2] > 0, got
    step(sim, orc, 5)
    return got


def full_rows(n=64):
    """Full rows: Alive records about unlisted members are dropped and counted; nothing is inserted, the view is not
    marked changed, and export still works."""
    from view_edit_scenarios import export_matches_oracle
    sim, orc = pair(n, 32, 32, seed=5)
    ev = crash_events(1, [7, 8, 9])  # (suspicions: records in flight for export)
    sim.inject(ev)
    orc.inject(ev)
    step(sim, orc, 3)
    got = join(sim, orc, [1, 2, 3], [40, 41, 42], where="full rows")
    assert got[1] == 0 and got[2] > 0, got
    assert export_matches_oracle(sim, orc) > 0


def refutations(n=80, **kw):
    """Joiners that are Suspect / Dead at their seeds: the seed's state carries the suspicion and the joiner refutes."""
    sim, orc = pair(n, 32, 12, seed=6, loss_ppm=30000, **kw)
    step(sim, orc, 2)
    vst = orc.get_array(A.ARR_VST).reshape(n, 32)
    vst[: n // 2, 0] = A.SUSPECT | (2 << 2)
    vst[n // 4: n // 2, 1] = A.DEAD
    for h in (sim, orc):
        h.set_array(A.ARR_VST, vst.reshape(-1))
    nbr = orc.get_array(A.ARR_NBR).reshape(n, 32)
    rows = np.arange(n // 2)
    before = orc.counters()[A.CTR_REFUTES]
    join(sim, orc, np.concatenate([nbr[rows, 0], nbr[n // 4: n // 2, 1]]),
         np.concatenate([rows, np.arange(n // 4, n // 2)]), where="refutations")
    assert orc.counters()[A.CTR_REFUTES] > before
    step(sim, orc, 3)


def save_join_load(n, rounds=8):
    """A join that changes no membership keeps the checkpoint: save -> join -> steps -> load -> the same again gives
    identical states. A fresh join that empties slots drops it."""
    from swim_b200._lib import SwimError
    sim, orc = pair(n, 32, 32, seed=7, loss_ppm=20000)
    step(sim, orc, 4)
    sim.save()
    nodes, seeds = np.arange(1, 40), np.arange(1, 40) * 7 % n
    keep = nodes != seeds
    nodes, seeds = nodes[keep], seeds[keep]
    got = join(sim, orc, nodes, seeds, where="before the replay")
    assert got[1] == 0
    step(sim, orc, rounds)
    first = sim.state()
    sim.load()
    assert sim.join(nodes, seeds) == got
    sim.step(rounds)
    again = sim.state()
    assert all(np.array_equal(first[k], again[k]) for k in first)
    sim.load()  # still valid
    sim.join([3], [9], fresh=True)
    with pytest.raises(SwimError) as e:
        sim.load()
    assert e.value.code == A.ESTATE


def export_after_join(n):
    """A fresh join that empties rows makes export refuse until the next step."""
    from swim_b200._lib import SwimError
    from view_edit_scenarios import export_matches_oracle
    sim, orc = pair(n, 32, 32, seed=8)
    step(sim, orc, 3)
    join(sim, orc, [4, 5], [6, 7], fresh=True, where="fresh")
    with pytest.raises(SwimError) as e:
        sim.export_round()
    assert e.value.code == A.ESTATE
    step(sim, orc, 1)
    export_matches_oracle(sim, orc)


def fresh_rebuild(n, frac=0.01, hosts=3, cap=32, deg=32, seed=9, rounds=(1, 9, 20)):
    """A fresh join of `frac` of the nodes through `hosts` seeds: the rows empty and refill, the next step rebuilds the
    mail graph, and the rounds after it match the oracle."""
    sim, orc = pair(n, cap, deg, seed=seed, loss_ppm=10000)
    step(sim, orc, 3, check=False)
    rng = np.random.default_rng(seed)
    nodes, seeds = restart_pairs(rng, n, rng.choice(n, size=hosts, replace=False), frac)
    got, want = sim.join(nodes, seeds, fresh=True), oracle_join(orc, nodes, seeds, fresh=True)
    assert got == want and got[1] > 0, (got, want)
    for a in (A.ARR_NBR, A.ARR_VST, A.ARR_VINC, A.ARR_VLAST, A.ARR_PB, A.ARR_PB_CNT, A.ARR_SELF_INC):
        assert np.array_equal(sim.get_array(a), orc.get_array(a)), A.ARRAY_NAMES[a]
    for c in rounds:
        step(sim, orc, c, check=False)
        assert sim.digest() == orc.digest(), f"digest differs at round {sim.round}"
        assert sim.counters().tolist() == orc.counters().tolist()
    sim.close()
    return got


def with_push_pull(n, cap=32, deg=12, seed=10):
    """push_pull and joins interleaved, with steps between them."""
    sim, orc = pair(n, cap, deg, seed=seed, loss_ppm=10000)
    rng = np.random.default_rng(seed)
    hosts = rng.choice(n, size=2, replace=False)
    for k in range(3):
        step(sim, orc, 4)
        got, want = sim.push_pull(), oracle_push_pull(orc)
        assert got == want
        nodes, seeds = restart_pairs(rng, n, hosts)
        join(sim, orc, nodes, seeds, fresh=k == 1, where=f"join {k}")
        got, want = sim.push_pull(), oracle_push_pull(orc)
        assert got == want
        assert_same_state(sim, orc, f"push_pull after join {k}")
    step(sim, orc, 5)


def error_paths(n=40):
    """SWIM_EINVAL on an id >= N or node == seed."""
    B.error_paths("join", ([1], [2]), [(nodes, seeds, True) for nodes, seeds in (([1, 2], [3, n]), ([n, 2], [3, 4]),
                                                                                ([1, 2], [3, 2]))], n)


sharded_not_connected = partial(B.sharded_not_connected, "join", ([30], [1], True))


# ------------------------------------------------------------------ sharded handles
def sharded_joins(world, n, mode, devices=None, rounds=24, every=6, **kw):
    """Joins through 3 seeds every `every` rounds on `world` ranks, alternately fresh and not, under events and loss.
    `kw` overrides config fields."""
    rng = np.random.default_rng(13)
    hosts = rng.choice(n, size=3, replace=False)
    B.sharded_every("join", lambda k: (*restart_pairs(rng, n, hosts), k % 2 == 1), world, n, mode, devices, rounds,
                    every, **kw)


def sharded_equals_single_shard(n, world, devices, mode="p2p", **kw):
    """A fresh join of 1 % of the nodes through 3 seeds, then a plain one."""
    B.sharded_equals_single_shard(
        "join", lambda rng, k: (*restart_pairs(rng, n, rng.choice(n, size=3, replace=False), 0.01), k == 0), n, world,
        devices, mode, **kw)
