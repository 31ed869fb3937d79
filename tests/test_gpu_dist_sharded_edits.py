"""Multi-GPU form of test_gpu_sharded_edits.py: one process per GPU (torchrun), over peer memory and through NCCL. A
sharded run with push_pull, remove_dead_nodes and add_members between its steps must give the single-shard oracle's
digests, totals, counters and state. Skipped below 2 GPUs."""
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import crash_events, default_config, generate_topology
from push_pull_oracle import push_pull as oracle_push_pull
from swim_b200 import _abi as A
from view_edit_scenarios import dead_entries, oracle_add, oracle_remove_dead

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = ["push_pull", "remove_dead_nodes", "add_members", "push_pull"]


def _gpus():
    import torch
    return torch.cuda.device_count()


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
@pytest.mark.parametrize("n", [1003, 65536])
def test_sharded_edits_equal_oracle(tmp_path, n, mode):
    world = min(_gpus(), 4)
    if world < 2:
        pytest.skip("needs 2 GPUs")
    from oracle.oracle import Oracle
    seed, loss = 77, 10000
    rng = np.random.default_rng(seed)
    nbr = generate_topology("random", n, 32, 16, seed=seed)
    events = crash_events(2, rng.choice(n, size=max(2, n // 20), replace=False))
    obs = rng.integers(0, n, size=max(64, n // 8))
    mem = (obs + rng.integers(1, n, size=len(obs))) % n
    rounds = [6, 8, 6, 10]
    np.savez(tmp_path / "case.npz", n=n, seed=seed, loss=loss, nbr=nbr, mode=mode, phases=np.array(PHASES),
             rounds=np.array(rounds), obs=obs, mem=mem, events=np.frombuffer(events.tobytes(), dtype=np.uint8))
    out = tmp_path / "result.npz"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29500 + os.getpid() % 2000),
           os.path.join(ROOT, "tests", "dist_sharded_edits_worker.py"), str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-6000:]
    got = np.load(out)
    ref = Oracle(default_config(n_nodes=n, k_indirect=3, fanout=4, pb_cap=6, suspicion_rounds=3, retransmit=5,
                                loss_ppm=loss, seed=seed))
    ref.set_view(nbr)
    ref.inject(events)
    digests = iter(got["digests"].tolist())
    for phase, rounds, total in zip(PHASES, rounds, got["totals"].tolist()):
        if phase == "push_pull":
            want = list(oracle_push_pull(ref))
        elif phase == "remove_dead_nodes":
            want = [dead_entries(ref), 0, 0]
            oracle_remove_dead(ref)
        else:
            want = list(oracle_add(ref, obs, mem, [1] * len(obs))) + [0]
        assert total == want, (phase, total, want)
        for c in (1, rounds - 1):
            ref.step(c)
            assert next(digests) == ref.digest(), f"digest differs at round {ref.round}"
    assert got["counters"].tolist() == ref.counters().tolist()
    assert int(got["mismatches"]) == ref.mismatches()
    for a in range(A.ARR_COUNT):
        assert np.array_equal(got[A.ARRAY_NAMES[a]], ref.get_array(a)), A.ARRAY_NAMES[a]
