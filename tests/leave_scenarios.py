"""Scenarios of the graceful leaves between steps (swim_sim_leave, DESIGN.md 2.8), shared by the emulator tests (small
sizes) and the H100 tests (2^16 nodes and up). Every call is checked against the CPU oracle's statement
(tests/between_steps_oracle.c, oracle_leave): both outputs, every state array, the counters, the digest and the mismatch
count, right after the call and after further steps. The sharded scenarios hold the shards' sums to the single-shard
oracle (between_steps_scenarios)."""
from functools import partial

import numpy as np

import between_steps_scenarios as B
from between_steps_scenarios import pair, step
from helpers import assert_same_state, crash_events, generate_topology, make_events, random_events
from swim_b200 import _abi as A

NM = A.NO_MEMBER
leave = partial(B.call, "leave")


def leave_list(rng, n, frac=0.03):
    """A share of the nodes, with some of them listed twice, in random order (down ones are ignored by the call)."""
    who = rng.choice(n, size=max(2, int(n * frac)), replace=False)
    return rng.permutation(np.concatenate([who, who[: max(1, len(who) // 4)]])).astype(np.uint32)


def leave_every(n, cap, deg, rounds=24, every=6, seed=1, **kw):
    """Steps with events (crashes, rejoins, injected records), churn and loss as given, and every `every` rounds a leave
    of 3 % of the nodes. Returns the summed outputs."""
    sim, orc = pair(n, cap, deg, seed=seed, **kw)
    rng = np.random.default_rng(seed)
    ev = random_events(rng, n, rounds, n_crash=max(2, n // 12), n_rejoin=max(1, n // 30), n_inject=max(1, n // 8))
    sim.inject(ev)
    orc.inject(ev)
    tot = np.zeros(2, dtype=np.int64)
    for _ in range(0, rounds, every):
        step(sim, orc, every, check=False)
        tot += leave(sim, orc, leave_list(rng, n), where=f"n={n} cap={cap} round {sim.round}")
    step(sim, orc, 2)
    sim.close()
    assert tot[0] > 0 and tot[1] > 0, tot
    return tot


def rows_of(nbr_lists, n, cap):
    """An id matrix from per-row member lists (ascending, vacancies last)."""
    nbr = np.full((n, cap), NM, dtype=np.uint32)
    for i, r in enumerate(nbr_lists):
        r = sorted(set(int(x) for x in r) - {i})[:cap]
        nbr[i, : len(r)] = r
    return nbr.reshape(-1)


def edge_cases(n=120):
    """n = 0; repeated and down ids; two leavers that list each other; an empty-row leaver; recipients that do not list
    their leaver; a leaver whose only members are Dead at it."""
    rng = np.random.default_rng(2)
    lists = [rng.choice(n, size=8, replace=False) for _ in range(n)]
    lists[3] = []  # an empty row
    lists[10] = [11, 12, 13]
    lists[11] = [10, 14]  # 10 and 11 list each other
    lists[20] = [21, 22]
    nbr = rows_of(lists, n, 32)
    sim, orc = pair(n, 32, nbr=nbr, seed=2)
    ev = crash_events(1, [5, 40])
    sim.inject(ev)
    orc.inject(ev)
    step(sim, orc, 3)
    assert sim.leave([]) == (0, 0)
    assert_same_state(sim, orc, "n = 0")
    assert leave(sim, orc, [5, 40, 5], where="down ids only") == (0, 0)
    got = leave(sim, orc, [3, 3, 3], where="an empty-row leaver")
    assert got == (1, 0), got
    got = leave(sim, orc, [10, 11, 10], where="leavers that list each other")
    assert got == (2, 3), got  # 12, 13 from 10; 14 from 11; neither hears about the other
    # recipients that do not list their leaver get `Nothing`: their rows and buffers are unchanged
    vst = orc.get_array(A.ARR_VST).reshape(n, 32)
    vst[20, :2] = A.DEAD  # 20 holds both its members Dead: nobody hears from it
    for h in (sim, orc):
        h.set_array(A.ARR_VST, vst.reshape(-1))
    assert leave(sim, orc, [20], where="members all Dead") == (1, 0)
    m = next(int(x) for x in lists[30] if x not in lists[int(x)] and orc.get_array(A.ARR_ALIVE)[int(x)])
    before = {a: orc.get_array(a).reshape(n, -1)[m].copy() for a in (A.ARR_NBR, A.ARR_VST, A.ARR_PB_CNT)}
    assert 30 not in before[A.ARR_NBR]
    leave(sim, orc, [30], where="a recipient that does not list the leaver")
    for a, v in before.items():
        assert np.array_equal(orc.get_array(a).reshape(n, -1)[m], v), A.ARRAY_NAMES[a]
    step(sim, orc, 4)


def hub(n, leavers, cap=32, deg=8, seed=4):
    """Many leavers that all list one hub, which lists some of them: the hub receives one record per leaver, its buffer
    overflows (PB_DROPPED), the ones it does not list are `Nothing`; then rounds."""
    rng = np.random.default_rng(seed)
    h = int(rng.integers(0, n))
    who = rng.choice(np.delete(np.arange(n), h), size=leavers, replace=False)
    nbr = generate_topology("random", n, cap, deg, seed=seed).reshape(n, cap).copy()
    row = np.sort(np.append(who[: cap // 2], np.delete(nbr[h], np.flatnonzero(nbr[h] == NM))))
    row = np.unique(row[row != h])[:cap]
    nbr[h] = NM
    nbr[h, : len(row)] = row
    for i in who:  # the hub replaces the member with the largest id (the row stays ascending, without i)
        r = nbr[i][nbr[i] != NM]
        if h not in r:
            r = np.sort(np.append(r[:-1], h)) if len(r) == cap else np.sort(np.append(r, h))
        nbr[i] = NM
        nbr[i, : len(r)] = r
    sim, orc = pair(n, cap, nbr=nbr.reshape(-1), seed=seed, loss_ppm=10000)
    step(sim, orc, 2)
    dropped = orc.counters()[A.CTR_PB_DROPPED]
    got = leave(sim, orc, who, where="hub")
    assert got[0] == leavers and got[1] >= leavers, got
    assert orc.counters()[A.CTR_PB_DROPPED] > dropped
    step(sim, orc, 5)
    sim.close()
    return got


def rejoin_after_leave(n=100, **kw):
    """A REJOIN event after a leave restarts the leaver with self_inc + 1; the Dead it left behind is refuted and the
    members learn it Alive again."""
    sim, orc = pair(n, 32, 12, seed=6, **kw)
    step(sim, orc, 3)
    who = [7, 8, 9]
    inc = orc.get_array(A.ARR_SELF_INC)[who].copy()
    got = leave(sim, orc, who, where="before the rejoin")
    assert got[0] == 3 and got[1] > 0
    ev = make_events(np.full(3, sim.round + 2, np.uint32), np.array(who, np.uint32), np.full(3, A.EV_REJOIN, np.uint8))
    sim.inject(ev)
    orc.inject(ev)
    step(sim, orc, 4)
    assert orc.get_array(A.ARR_ALIVE)[who].all()
    assert (orc.get_array(A.ARR_SELF_INC)[who] > inc).all()
    step(sim, orc, 20)
    sim.close()


def churn_rejoin_then_leave(n=200):
    """A node that the seeded churn crashed, that a REJOIN event brings back before its churn rejoin round and that then
    leaves: back_at is cleared, so it stays down past that round."""
    sim, orc = pair(n, 32, 12, seed=7, churn_ppm=20000, rejoin_min=20, rejoin_max=30)
    step(sim, orc, 4)
    back = orc.get_array(A.ARR_BACK_AT)
    alive = orc.get_array(A.ARR_ALIVE)
    who = np.flatnonzero((alive == 0) & (back > sim.round + 3))[:3]
    assert len(who), "no churn crash"
    ev = make_events(np.full(len(who), sim.round + 1, np.uint32), who.astype(np.uint32),
                     np.full(len(who), A.EV_REJOIN, np.uint8))
    sim.inject(ev)
    orc.inject(ev)
    step(sim, orc, 1)
    assert orc.get_array(A.ARR_ALIVE)[who].all() and (orc.get_array(A.ARR_BACK_AT)[who] == back[who]).all()
    got = leave(sim, orc, who, where="after an early rejoin")
    assert got[0] == len(who)
    assert not orc.get_array(A.ARR_BACK_AT)[who].any()
    step(sim, orc, int(back[who].max()) - sim.round + 2)
    assert not sim.get_array(A.ARR_ALIVE)[who].any()
    sim.close()


def save_leave_load(n, rounds=8):
    """A leave keeps the checkpoint: save -> leave -> steps -> load -> the same again gives identical states."""
    sim, orc = pair(n, 32, 32, seed=7, loss_ppm=20000)
    step(sim, orc, 4)
    sim.save()
    who = np.arange(1, n, max(2, n // 40))
    got = leave(sim, orc, who, where="before the replay")
    step(sim, orc, rounds)
    first = sim.state()
    sim.load()
    assert sim.leave(who) == got
    sim.step(rounds)
    again = sim.state()
    assert all(np.array_equal(first[k], again[k]) for k in first)
    sim.load()  # still valid
    sim.close()


def export_after_leave(n):
    """swim_sim_export_round keeps working after a leave; the next round's export equals the oracle's envelopes."""
    from view_edit_scenarios import export_matches_oracle
    sim, orc = pair(n, 32, 32, seed=8)
    step(sim, orc, 3)
    leave(sim, orc, [4, 5, 6], where="export")
    export_matches_oracle(sim, orc)
    step(sim, orc, 1)
    assert export_matches_oracle(sim, orc) > 0
    sim.close()


def with_push_pull_and_join(n, cap=32, deg=12, seed=10):
    """Leaves, push_pull and joins interleaved, with steps between them."""
    from between_steps_oracle import join as oracle_join, push_pull as oracle_push_pull
    from join_scenarios import restart_pairs
    sim, orc = pair(n, cap, deg, seed=seed, loss_ppm=10000)
    rng = np.random.default_rng(seed)
    hosts = rng.choice(n, size=2, replace=False)
    for k in range(3):
        step(sim, orc, 4)
        leave(sim, orc, leave_list(rng, n, 0.02), where=f"leave {k}")
        assert sim.push_pull() == oracle_push_pull(orc)
        assert_same_state(sim, orc, f"push_pull after leave {k}")
        nodes, seeds = restart_pairs(rng, n, hosts)
        assert sim.join(nodes, seeds, k == 1) == oracle_join(orc, nodes, seeds, k == 1)
        leave(sim, orc, leave_list(rng, n, 0.02), where=f"leave after join {k}")
    step(sim, orc, 5)
    sim.close()


def error_paths(n=40):
    """SWIM_EINVAL on an id >= N."""
    B.error_paths("leave", ([1],), [([1, 2, n],), ([n + 5],), ([0xFFFFFFFF, 3],)], n)


sharded_not_connected = partial(B.sharded_not_connected, "leave", ([30],))


# ------------------------------------------------------------------ sharded handles
def sharded_leaves(world, n, mode, devices=None, rounds=24, every=6, **kw):
    """A leave of 3 % of the nodes every `every` rounds on `world` ranks, under events and loss. `kw` overrides config
    fields."""
    rng = np.random.default_rng(13)
    B.sharded_every("leave", lambda k: (leave_list(rng, n),), world, n, mode, devices, rounds, every, **kw)


def sharded_equals_single_shard(n, world, devices, mode="p2p", **kw):
    """Two leaves of 1 % of the nodes."""
    B.sharded_equals_single_shard("leave", lambda rng, k: (leave_list(rng, n, 0.01),), n, world, devices, mode, **kw)


def suspect_turned_dead(n=60, suspicion_max=0):
    """Recipients that hold the leaver Suspect: its Dead turns the entry Dead (countdown and confirmations gone)."""
    sim, orc = pair(n, 32, 32, "ring", seed=3, suspicion_max=suspicion_max)
    step(sim, orc, 2)
    L = 17
    nbr = orc.get_array(A.ARR_NBR).reshape(n, 32)
    vst = orc.get_array(A.ARR_VST).reshape(n, 32)
    rows, slots = np.nonzero(nbr == L)
    vst[rows, slots] = A.SUSPECT | (2 << 2)
    for h in (sim, orc):
        h.set_array(A.ARR_VST, vst.reshape(-1))
    got = leave(sim, orc, [L], where="Suspect holders")
    assert got[0] == 1 and got[1] > 0
    after = orc.get_array(A.ARR_VST).reshape(n, 32)[rows, slots] & 3
    assert (after == A.DEAD).sum() == got[1], (after, got)
    step(sim, orc, 3)
    sim.close()
