"""The bulk membership calls and push-pull on sharded handles, on the H100: world 2 and 4 with every rank's handle in this
process and on device 0, connected over peer memory (raw device pointers), against the single-shard oracle after every
call and every chunk of rounds. Shards stay small for the scenarios with rounds: every rank's round kernel must be
resident at the same time (test_gpu_shards_one_device.py explains why). The larger check runs no rounds. The emulator
versions are in test_emu_sharded_edits.py; test_gpu_dist_sharded_edits.py is the multi-GPU form."""
import pytest

import sharded_edit_scenarios as S
from swim_b200 import _abi as A

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def fused_exchange(monkeypatch):
    monkeypatch.setenv("SWIM_ROUND_KERNEL", "1")


def dev(world):
    return [0] * world


@pytest.mark.parametrize("world", [2, 4])
def test_remove_dead_nodes(world):
    S.remove_dead_then_rounds(world, 1201, "p2p", devices=dev(world), chunks=(1, 1, 6, 20))


@pytest.mark.parametrize("world,min_age", [(2, 7), (4, 1)])
def test_remove_dead_nodes_min_age(world, min_age):
    S.remove_dead_min_age(world, 1000, "p2p", min_age, devices=dev(world))


@pytest.mark.parametrize("world", [2, 4])
def test_add_members(world):
    S.add_members_then_rounds(world, 1202, "p2p", devices=dev(world), chunks=(1, 3, 16))


@pytest.mark.parametrize("world", [2, 4])
def test_push_pull_inserts_then_rounds(world):
    S.push_pull_inserts_then_rounds(world, 1203, "p2p", devices=dev(world))


@pytest.mark.parametrize("world,flags,churn,smax", [
    (2, 0, (20000, 3, 8), 0),
    (4, A.F_STRICT_OVERRIDE, None, 0),
    (2, 0, None, 9),
    (4, A.F_STRICT_OVERRIDE | A.F_ROUND_ROBIN, (30000, 2, 6), 8),
])
def test_push_pull_every(world, flags, churn, smax):
    S.push_pull_every(world, 1100, "p2p", rounds=60, every=12, devices=dev(world), flags=flags, churn=churn,
                      suspicion_max=smax)


@pytest.mark.parametrize("world", [2, 4])
def test_edit_save_load(world):
    S.edit_save_load(world, 1000, "p2p", devices=dev(world))


def test_tiny_last_shard():
    S.tiny_last_shard(4, 13, "p2p", devices=dev(4))  # shards of 4, 4, 4 and 1 rows


def test_scalar_insert_still_refused():
    S.scalar_insert_refused(2, 600, "p2p", devices=dev(2))


def test_large_view_equals_single_shard():
    S.large_equals_single_shard(1 << 18, 2, dev(2))
