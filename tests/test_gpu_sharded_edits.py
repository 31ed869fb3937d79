"""The bulk membership calls and push-pull on sharded handles, on the H100: world 2 and 4 with every rank's handle in this
process and on device 0, connected over peer memory (raw device pointers) and, as "nccl" cases, through the staged
exchange with the in-process NCCL stand-in (tests/nccl_fixtures.py), against the single-shard oracle after every call and
every chunk of rounds. Shards stay small for the scenarios with rounds: over peer memory every rank's round kernel must
be resident at the same time (test_gpu_shards_one_device.py explains why). The larger check runs no rounds. The emulator
versions are in test_emu_sharded_edits.py; test_gpu_dist_between_steps.py is the multi-GPU form."""
import pytest

import sharded_edit_scenarios as S
from nccl_fixtures import fake_nccl_gpu, fake_nccl_gpu_lib, staged_too  # noqa: F401  (fixtures)
from swim_b200 import _abi as A

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def fused_exchange(monkeypatch):
    monkeypatch.setenv("SWIM_ROUND_KERNEL", "1")


@pytest.fixture
def mode(request):
    """The exchange of a case: "p2p", or "nccl" with the stand-in bound."""
    if request.param == "nccl":
        request.getfixturevalue("fake_nccl_gpu")
    return request.param


def dev(world):
    return [0] * world


@pytest.mark.parametrize("world,mode", staged_too([2, 4], ["2", "4"]), indirect=["mode"])
def test_remove_dead_nodes(world, mode):
    S.remove_dead_then_rounds(world, 1201, mode, devices=dev(world), chunks=(1, 1, 6, 20))


@pytest.mark.parametrize("world,min_age,mode", staged_too([(2, 7), (4, 1)], ["2-7", "4-1"]), indirect=["mode"])
def test_remove_dead_nodes_min_age(world, min_age, mode):
    S.remove_dead_min_age(world, 1000, mode, min_age, devices=dev(world))


@pytest.mark.parametrize("world,mode", staged_too([2, 4], ["2", "4"]), indirect=["mode"])
def test_add_members(world, mode):
    S.add_members_then_rounds(world, 1202, mode, devices=dev(world), chunks=(1, 3, 16))


@pytest.mark.parametrize("world,mode", staged_too([2, 4], ["2", "4"]), indirect=["mode"])
def test_push_pull_inserts_then_rounds(world, mode):
    S.push_pull_inserts_then_rounds(world, 1203, mode, devices=dev(world))


@pytest.mark.parametrize("world,flags,churn,smax,mode", staged_too([
    (2, 0, (20000, 3, 8), 0),
    (4, A.F_STRICT_OVERRIDE, None, 0),
    (2, 0, None, 9),
    (4, A.F_STRICT_OVERRIDE | A.F_ROUND_ROBIN, (30000, 2, 6), 8),
], ["2-0-churn0-0", "4-1-None-0", "2-0-None-9", "4-3-churn3-8"]), indirect=["mode"])
def test_push_pull_every(world, flags, churn, smax, mode):
    S.push_pull_every(world, 1100, mode, rounds=60, every=12, devices=dev(world), flags=flags, churn=churn,
                      suspicion_max=smax)


@pytest.mark.parametrize("world,mode", staged_too([2, 4], ["2", "4"]), indirect=["mode"])
def test_edit_save_load(world, mode):
    S.edit_save_load(world, 1000, mode, devices=dev(world))


def test_tiny_last_shard():
    S.tiny_last_shard(4, 13, "p2p", devices=dev(4))  # shards of 4, 4, 4 and 1 rows


def test_scalar_insert_still_refused():
    S.scalar_insert_refused(2, 600, "p2p", devices=dev(2))


def test_large_view_equals_single_shard():
    S.large_equals_single_shard(1 << 18, 2, dev(2))
