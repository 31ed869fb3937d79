"""Multi-GPU form of the sharded leave tests: one process per GPU (torchrun), over peer memory and through NCCL. A
sharded run with graceful leaves between its steps must give the single-shard oracle's totals, digests, counters and
state. Skipped below 2 GPUs."""
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import crash_events, default_config, generate_topology
from leave_oracle import leave as oracle_leave
from leave_scenarios import leave_list
from swim_b200 import _abi as A

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gpus():
    import torch
    return torch.cuda.device_count()


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
@pytest.mark.parametrize("n", [1003, 65536])
def test_sharded_leaves_equal_oracle(tmp_path, n, mode):
    world = min(_gpus(), 4)
    if world < 2:
        pytest.skip("needs 2 GPUs")
    from oracle.oracle import Oracle
    seed, loss = 78, 10000
    rng = np.random.default_rng(seed)
    nbr = generate_topology("random", n, 32, 16, seed=seed)
    events = crash_events(2, rng.choice(n, size=max(2, n // 20), replace=False))
    rounds = [6, 8, 6, 10]
    lists = [leave_list(rng, n, 0.02) for _ in rounds]
    case = dict(n=n, seed=seed, loss=loss, nbr=nbr, mode=mode, rounds=np.array(rounds),
                events=np.frombuffer(events.tobytes(), dtype=np.uint8))
    for k, ids in enumerate(lists):
        case[f"ids{k}"] = ids
    np.savez(tmp_path / "case.npz", **case)
    out = tmp_path / "result.npz"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29500 + os.getpid() % 2000),
           os.path.join(ROOT, "tests", "dist_leave_worker.py"), str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-6000:]
    got = np.load(out)
    ref = Oracle(default_config(n_nodes=n, k_indirect=3, fanout=4, pb_cap=6, suspicion_rounds=3, retransmit=5,
                                loss_ppm=loss, seed=seed))
    ref.set_view(nbr)
    ref.inject(events)
    for k, (c, ids) in enumerate(zip(rounds, lists)):
        ref.step(c)
        want = list(oracle_leave(ref, ids))
        assert got["totals"][k].tolist() == want, (k, got["totals"][k], want)
        ref.step(1)
        assert int(got["digests"][k]) == ref.digest(), f"digest differs at round {ref.round}"
    assert got["counters"].tolist() == ref.counters().tolist()
    assert int(got["mismatches"]) == ref.mismatches()
    for a in range(A.ARR_COUNT):
        assert np.array_equal(got[A.ARRAY_NAMES[a]], ref.get_array(a)), A.ARRAY_NAMES[a]
