"""Scenarios of the push-pull state exchange between steps (swim_sim_push_pull, DESIGN.md 2.6), shared by the emulator
tests (small sizes) and the H100 tests (2^16 nodes and up). Every call is checked against the CPU oracle: the three
outputs, every state array, the counters and the digest (between_steps_scenarios)."""
import numpy as np
import pytest

from between_steps_scenarios import call, error_paths as _error_paths, pair, step
from helpers import assert_same_state, crash_events, random_events
from swim_b200 import _abi as A


def push_pull(sim, orc, where):
    return call("push_pull", sim, orc, where=where)


def with_events(sim, orc, n, rounds, seed):
    ev = random_events(np.random.default_rng(seed), n, rounds, n_crash=max(2, n // 12), n_rejoin=max(1, n // 30),
                       n_inject=max(1, n // 8))
    sim.inject(ev)
    orc.inject(ev)


def step_push_pull_step(n, cap, deg, kind="random", rounds=30, every=6, seed=1, events=True, **kw):
    """Steps with events (crashes, rejoins, injected records), churn and loss as given, and a push_pull every `every`
    rounds. Returns the summed outputs."""
    sim, orc = pair(n, cap, deg, kind, seed, **kw)
    if events:
        with_events(sim, orc, n, rounds, seed)
    tot = np.zeros(3, dtype=np.int64)
    for r in range(0, rounds, every):
        step(sim, orc, every, check=False)
        tot += push_pull(sim, orc, f"{kind} n={n} cap={cap} round {sim.round}")
    step(sim, orc, 2)
    return sim, orc, tot


def no_partner_cases(n=24):
    """A node with no Alive slot picks nobody, a crashed partner exchanges nothing, a crashed node neither sends nor
    receives; and everybody down gives zero exchanges."""
    sim, orc = pair(n, 32, 3, "ring", seed=2)
    ev = crash_events(1, [1, 2, 3, 23, 22, 21, 10])  # 0 and 11.. lose their neighbours
    sim.inject(ev)
    orc.inject(ev)
    step(sim, orc, 12)
    push_pull(sim, orc, "crashed partners")
    sim2, orc2 = pair(8, 32, 32, "complete", seed=3)
    ev = crash_events(1, list(range(8)))
    sim2.inject(ev)
    orc2.inject(ev)
    step(sim2, orc2, 1)
    assert push_pull(sim2, orc2, "everybody down") == (0, 0, 0)


def same_round_same_partners(n, cap=32, deg=32):
    """Two calls at one round pick the same partners: with full rows and no changes to pick up, the second call sees the
    same exchanges."""
    sim, orc = pair(n, cap, deg, "random", seed=4)
    a = push_pull(sim, orc, "first")
    b = push_pull(sim, orc, "second, same round")
    assert a[0] == b[0] > 0


def save_push_pull_load(n, cap=32, rounds=12):
    """Full rows (no inserts): the checkpoint survives push_pull, and save -> push_pull -> steps -> load -> the same
    again gives identical states."""
    sim, orc = pair(n, cap, cap, "random", seed=5, loss_ppm=20000)
    with_events(sim, orc, n, 6, seed=5)
    step(sim, orc, 6)
    sim.save()
    got = push_pull(sim, orc, "before the checkpoint's replay")
    assert got[1] == 0
    step(sim, orc, rounds)
    first = sim.state()
    sim.load()
    assert sim.push_pull() == got
    sim.step(rounds)
    again = sim.state()
    assert all(np.array_equal(first[k], again[k]) for k in first)
    sim.load()  # the checkpoint is still valid
    return sim, orc


def inserts_then_rounds(n, cap=32, deg=12, rounds=50, chunk=10, kind="random", seed=6):
    """Random views with D < cap: push_pull inserts members; the next step rebuilds the mail graph, and the rounds after
    it stay equal to the oracle."""
    from swim_b200._lib import SwimError
    sim, orc = pair(n, cap, deg, kind, seed=seed, loss_ppm=10000)
    ev = crash_events(2, np.random.default_rng(seed).choice(n, size=max(1, n // 25), replace=False))
    sim.inject(ev)
    orc.inject(ev)
    step(sim, orc, 4)
    sim.save()
    got = push_pull(sim, orc, "inserts")
    assert got[1] > 0, got
    with pytest.raises(SwimError) as e:  # the checkpoint belongs to the old view
        sim.load()
    assert e.value.code == A.ESTATE
    for _ in range(0, rounds, chunk):
        step(sim, orc, chunk)
    return sim, orc, got


def full_rows_drop_inserts(n=40):
    """Rows filled to the cap: an Alive record about an unlisted member is dropped and counted."""
    sim, orc = pair(n, 32, 32, "random", seed=7)
    got = push_pull(sim, orc, "full rows")
    assert got[2] > 0 and got[1] == 0, got


def push_pull_then_edits(n, cap=32, deg=16):
    """push_pull (with inserts), then remove_dead_nodes and add_members, then steps."""
    from view_edit_scenarios import oracle_add, oracle_remove_dead
    sim, orc = pair(n, cap, deg, "random", seed=8)
    ev = crash_events(2, np.random.default_rng(8).choice(n, size=max(2, n // 10), replace=False))
    sim.inject(ev)
    orc.inject(ev)
    step(sim, orc, 10)
    assert push_pull(sim, orc, "before the edits")[1] > 0
    sim.remove_dead_nodes()
    oracle_remove_dead(orc)
    rng = np.random.default_rng(9)
    obs = rng.integers(0, n, size=n // 2)
    mem = (obs + 1 + rng.integers(0, n - 1, size=n // 2)) % n
    assert sim.add_members(obs, mem, 1) == oracle_add(orc, obs, mem, [1] * len(obs))
    assert_same_state(sim, orc, "after the edits")
    for _ in range(4):
        step(sim, orc, 3)
    push_pull(sim, orc, "after the edits and steps")
    step(sim, orc, 5)


def export_after_push_pull(n):
    """Without inserts the last round's envelopes still stand (export works); with inserts export refuses until the next
    step."""
    from swim_b200._lib import SwimError
    from view_edit_scenarios import export_matches_oracle
    sim, orc = pair(n, 32, 32, "random", seed=10)
    with_events(sim, orc, n, 5, seed=10)
    step(sim, orc, 5)
    assert push_pull(sim, orc, "full rows")[1] == 0
    assert export_matches_oracle(sim, orc) > 0
    sim, orc = pair(n, 32, 10, "random", seed=11)
    step(sim, orc, 3)
    assert push_pull(sim, orc, "inserts")[1] > 0
    with pytest.raises(SwimError) as e:
        sim.export_round()
    assert e.value.code == A.ESTATE
    step(sim, orc, 1)
    export_matches_oracle(sim, orc)


def error_paths(n=40):
    _error_paths("push_pull", (), n=n)
