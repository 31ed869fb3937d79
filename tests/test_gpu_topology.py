"""The device view generator (swim_sim_generate_view) on the GPU: every kind bit-identical to the host generator at 2^16
and 2^20 nodes (the complete view at its largest size, 257 nodes on 256 slots), random and symmetric views at 2^22, a
C3-size run on symmetric views against the oracle, and world 2 on one device against one shard."""
import pytest

import topology_scenarios as T

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kind", ["ring", "random", "symmetric"])
@pytest.mark.parametrize("log_n", [16, 20])
def test_device_matrix_equals_host(kind, log_n):
    T.device_equals_host(kind, (1 << log_n) + 3, 32, 32, 0x5EED0000 + log_n, full_state=log_n == 16, steps=3)


@pytest.mark.parametrize("kind", ["random", "symmetric"])
def test_device_matrix_equals_host_2_22(kind):
    T.device_equals_host(kind, 1 << 22, 32, 32, 7, full_state=False)


@pytest.mark.parametrize("kind,cap,deg", [("complete", 256, 0), ("symmetric", 256, 256), ("random", 64, 48), ("ring", 128, 100)])
def test_wide_rows_equal_host(kind, cap, deg):
    T.device_equals_host(kind, 257 if kind == "complete" else 40000, cap, deg, 11, steps=3)


def test_c3_size_run_on_symmetric_views():
    """BASELINE config C3's size and burst (N = 1,048,576, 1,048 crashes at round 10) on symmetric views generated on the
    device: digest, counters and convergence count equal to the oracle's through 30 rounds, every array at the end."""
    T.symmetric_run_equals_oracle(1 << 20, 32, rounds=30, chunks=[1] * 12 + [8, 10], crashes=1048, seed=0x5EED0001 + 3)


def test_world_2_on_one_device_equals_single():
    T.sharded_equals_single(2, "symmetric", (1 << 18) + 1, 32, 5, devices=[0, 0])


def test_errors_and_checkpoint():
    T.errors_and_checkpoint(1 << 16)
