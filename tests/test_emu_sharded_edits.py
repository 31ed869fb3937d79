"""The bulk membership calls and push-pull on sharded handles, on the SIMT emulator (tests/emu): world 2 and 3, over
peer memory and through the staged NCCL exchange (tests/emu/fake_nccl.cpp), against the single-shard oracle after every
call and every chunk of rounds. The H100 versions are in test_gpu_sharded_edits.py."""
import pytest

import sharded_edit_scenarios as S
from swim_b200 import _abi as A
from emu_fixtures import emu_library, fake_nccl  # noqa: F401  (autouse fixtures)

MODES = ["p2p", "nccl"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("world", [2, 3])
def test_remove_dead_nodes(world, mode):
    S.remove_dead_then_rounds(world, 241, mode)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("world,min_age", [(2, 7), (3, 1)])
def test_remove_dead_nodes_min_age(world, min_age, mode):
    S.remove_dead_min_age(world, 250, mode, min_age)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("world", [2, 3])
def test_add_members(world, mode):
    S.add_members_then_rounds(world, 262, mode)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("world", [2, 3])
def test_push_pull_inserts_then_rounds(world, mode):
    S.push_pull_inserts_then_rounds(world, 203, mode)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("world,flags,churn,smax", [
    (2, 0, (20000, 3, 8), 0),
    (3, A.F_STRICT_OVERRIDE, None, 0),
    (3, 0, None, 9),
    (2, A.F_STRICT_OVERRIDE | A.F_ROUND_ROBIN, (30000, 2, 6), 8),
])
def test_push_pull_every(world, flags, churn, smax, mode):
    S.push_pull_every(world, 230, mode, flags=flags, churn=churn, suspicion_max=smax)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("world", [2, 3])
def test_edit_save_load(world, mode):
    S.edit_save_load(world, 200, mode)


@pytest.mark.parametrize("mode", MODES)
def test_tiny_last_shard(mode):
    S.tiny_last_shard(3, 7, mode)


@pytest.mark.parametrize("mode", MODES)
def test_scalar_insert_still_refused(mode):
    S.scalar_insert_refused(2, 120, mode)


def test_not_connected_refused():
    S.not_connected_refused()
