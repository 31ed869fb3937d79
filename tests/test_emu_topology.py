"""The device view generator (swim_sim_generate_view) on the SIMT emulator (tests/emu): every kind bit-identical to the
host generator, sharded handles equal to one shard, and a run on symmetric views equal to the oracle. The H100 versions
of these scenarios are in test_gpu_topology.py."""
import pytest

import topology_scenarios as T
from emu_fixtures import emu_library  # noqa: F401  (autouse fixtures)


@pytest.mark.parametrize("kind,n,cap,deg,seed", [
    ("complete", 1, 32, 0, 1), ("complete", 30, 32, 0, 1), ("complete", 33, 32, 0, 2), ("complete", 129, 128, 0, 3),
    ("ring", 1, 32, 0, 1), ("ring", 3, 32, 2, 1), ("ring", 5, 32, 4, 1), ("ring", 33, 32, 32, 1), ("ring", 150, 32, 9, 1),
    ("ring", 301, 64, 60, 1), ("ring", 257, 256, 256, 1),
    ("random", 2, 32, 1, 4), ("random", 33, 32, 32, 5), ("random", 301, 32, 24, 6), ("random", 150, 64, 50, 2 ** 33 + 7),
    ("random", 259, 256, 200, 8),
    ("symmetric", 3, 32, 2, 1), ("symmetric", 5, 32, 4, 9), ("symmetric", 33, 32, 32, 10), ("symmetric", 301, 32, 32, 11),
    ("symmetric", 150, 64, 20, 2 ** 40 + 3), ("symmetric", 257, 256, 256, 12), ("symmetric", 1023, 128, 64, 13),
])
def test_device_matrix_equals_host(kind, n, cap, deg, seed):
    T.device_equals_host(kind, n, cap, deg, seed, steps=4 if n > 2 else 0)


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("kind", ["random", "symmetric"])
def test_sharded_equals_single(world, kind):
    T.sharded_equals_single(world, kind, 301, 24, 6)


def test_symmetric_run_equals_oracle():
    T.symmetric_run_equals_oracle(307, 24, rounds=30, chunks=[1] * 12 + [8, 10], crashes=12, churn=(20000, 3, 8), loss=20000)


def test_errors_and_checkpoint():
    T.errors_and_checkpoint(100)
