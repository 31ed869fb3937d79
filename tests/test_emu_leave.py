"""Graceful leaves (swim_sim_leave) on the SIMT emulator (tests/emu), against the oracle after every call: single-shard
scenarios at every row width, and sharded handles of world 2, 3 and 4 over peer memory and through the staged NCCL
exchange (tests/emu/fake_nccl.cpp). The H100 versions are in test_gpu_leave.py."""
import os

import pytest

import leave_scenarios as S
from swim_b200 import _abi as A
from emu_fixtures import emu_library, fake_nccl  # noqa: F401  (autouse fixtures)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("cap", [32, 64, 128, 256])
def test_every_row_width(cap):
    S.leave_every(160, cap, min(cap // 2 + 3, 100), rounds=18, every=6, seed=cap, loss_ppm=20000, churn_ppm=5000,
                  rejoin_min=2, rejoin_max=6)


@pytest.mark.parametrize("flags,suspicion_max", [(A.F_STRICT_OVERRIDE, 0), (0, 9), (A.F_ROUND_ROBIN, 0)])
def test_protocol_variants(flags, suspicion_max):
    S.leave_every(140, 32, 14, rounds=24, every=4, flags=flags, suspicion_max=suspicion_max, loss_ppm=30000)


def test_edge_cases():
    S.edge_cases()


def test_hub():
    S.hub(600, 300)


def test_rejoin_after_leave():
    S.rejoin_after_leave()


def test_churn_rejoin_then_leave():
    S.churn_rejoin_then_leave()


def test_save_leave_load():
    S.save_leave_load(160)


def test_export_after_leave():
    S.export_after_leave(80)


def test_with_push_pull_and_join():
    S.with_push_pull_and_join(200)


def test_error_paths():
    S.error_paths()
    S.sharded_not_connected()


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
@pytest.mark.parametrize("world", [2, 3, 4])
def test_sharded(world, mode):
    S.sharded_leaves(world, 211, mode)


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
def test_sharded_equals_single_shard(mode):
    S.sharded_equals_single_shard(700, 3, None, mode)


@pytest.mark.parametrize("suspicion_max", [0, 9])
def test_suspect_turned_dead(suspicion_max):
    S.suspect_turned_dead(suspicion_max=suspicion_max)
