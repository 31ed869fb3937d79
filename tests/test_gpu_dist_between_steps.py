"""Multi-GPU form of the sharded tests of the calls between steps: one process per GPU (torchrun), over peer memory and
through NCCL. A sharded run with membership edits (push_pull, remove_dead_nodes, add_members), with seed joins
(alternately fresh and not) or with graceful leaves between its steps must give the single-shard oracle's totals,
digests, counters and state. Skipped below 2 GPUs."""
import os
import subprocess
import sys

import numpy as np
import pytest

import between_steps_oracle
from helpers import crash_events, default_config, generate_topology
from join_scenarios import restart_pairs
from leave_scenarios import leave_list
from swim_b200 import _abi as A
from view_edit_scenarios import dead_entries, oracle_add, oracle_remove_dead

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROUNDS = [6, 8, 6, 10]


def _gpus():
    import torch
    return torch.cuda.device_count()


# A case's phases, drawn from its generator after the crash events: (rounds before the call, call, its arguments, the
# chunks of rounds after it, each followed by a digest).
def edits(rng, n):
    obs = rng.integers(0, n, size=max(64, n // 8))
    mem = (obs + rng.integers(1, n, size=len(obs))) % n
    calls = [("push_pull", ()), ("remove_dead_nodes", ()), ("add_members", (obs, mem, 1)), ("push_pull", ())]
    return [(0, call, args, [1, r - 1]) for (call, args), r in zip(calls, ROUNDS)]


def joins(rng, n):
    hosts = rng.choice(n, size=3, replace=False)
    return [(r, "join", (*restart_pairs(rng, n, hosts, 0.02), fresh), [1])
            for r, fresh in zip(ROUNDS, [False, True, False, True])]


def leaves(rng, n):
    return [(r, "leave", (leave_list(rng, n, 0.02),), [1]) for r in ROUNDS]


CASES = {"edits": (77, edits), "joins": (78, joins), "leaves": (78, leaves)}


def oracle_call(ref, call, args):
    """The call's totals on the oracle, as the worker pads them."""
    if call == "remove_dead_nodes":
        want = [dead_entries(ref)]
        oracle_remove_dead(ref)
    elif call == "add_members":
        obs, mem, inc = args
        want = list(oracle_add(ref, obs, mem, [inc] * len(obs)))
    else:
        want = list(getattr(between_steps_oracle, call)(ref, *args))
    return want + [0] * (3 - len(want))


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
@pytest.mark.parametrize("n", [1003, 65536])
@pytest.mark.parametrize("case", list(CASES))
def test_sharded_calls_equal_oracle(tmp_path, case, n, mode):
    world = min(_gpus(), 4)
    if world < 2:
        pytest.skip("needs 2 GPUs")
    from oracle.oracle import Oracle
    seed, loss = CASES[case][0], 10000
    rng = np.random.default_rng(seed)
    nbr = generate_topology("random", n, 32, 16, seed=seed)
    events = crash_events(2, rng.choice(n, size=max(2, n // 20), replace=False))
    phases = CASES[case][1](rng, n)
    spec = dict(n=n, seed=seed, loss=loss, nbr=nbr, mode=mode, events=np.frombuffer(events.tobytes(), dtype=np.uint8),
                before=np.array([p[0] for p in phases]), calls=np.array([p[1] for p in phases]),
                nargs=np.array([len(p[2]) for p in phases]), after=np.array([p[3] + [0] * (2 - len(p[3])) for p in phases]))
    for k, (_, _, args, _) in enumerate(phases):
        for i, a in enumerate(args):
            spec[f"arg{k}_{i}"] = a
    np.savez(tmp_path / "case.npz", **spec)
    out = tmp_path / "result.npz"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29500 + os.getpid() % 2000),
           os.path.join(ROOT, "tests", "dist_between_steps_worker.py"), str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-6000:]
    got = np.load(out)
    ref = Oracle(default_config(n_nodes=n, k_indirect=3, fanout=4, pb_cap=6, suspicion_rounds=3, retransmit=5,
                                loss_ppm=loss, seed=seed))
    ref.set_view(nbr)
    ref.inject(events)
    digests = iter(got["digests"].tolist())
    for k, (before, call, args, after) in enumerate(phases):
        if before:
            ref.step(before)
        want = oracle_call(ref, call, args)
        assert got["totals"][k].tolist() == want, (k, call, got["totals"][k], want)
        for c in after:
            ref.step(c)
            assert next(digests) == ref.digest(), f"digest differs at round {ref.round}"
    assert next(digests, None) is None
    assert got["counters"].tolist() == ref.counters().tolist()
    assert int(got["mismatches"]) == ref.mismatches()
    for a in range(A.ARR_COUNT):
        assert np.array_equal(got[A.ARRAY_NAMES[a]], ref.get_array(a)), A.ARRAY_NAMES[a]
