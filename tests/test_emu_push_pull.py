"""The push-pull state exchange (swim_sim_push_pull) on the SIMT emulator (tests/emu), against the oracle after every
call. The H100 versions of these scenarios are in test_gpu_push_pull.py."""
import pytest

import push_pull_scenarios as S
from swim_b200 import _abi as A
from emu_fixtures import emu_library  # noqa: F401  (autouse fixtures)


@pytest.mark.parametrize("cap", [32, 64, 128, 256])
def test_every_row_width(cap):
    S.step_push_pull_step(160, cap, min(cap // 2 + 3, 100), rounds=18, every=6, seed=cap)


@pytest.mark.parametrize("kind,deg", [("ring", 4), ("complete", 32), ("random", 20)])
def test_step_push_pull_step_with_churn_and_loss(kind, deg):
    n = 33 if kind == "complete" else 150
    _, _, tot = S.step_push_pull_step(n, 32, deg, kind, rounds=30, every=5, loss_ppm=20000, churn_ppm=5000,
                                      rejoin_min=2, rejoin_max=6)
    assert tot[0] > 0


@pytest.mark.parametrize("flags,suspicion_max", [(A.F_STRICT_OVERRIDE, 0), (0, 9), (A.F_ROUND_ROBIN, 0)])
def test_protocol_variants(flags, suspicion_max):
    S.step_push_pull_step(140, 32, 14, rounds=24, every=4, flags=flags, suspicion_max=suspicion_max, loss_ppm=30000)


def test_small_piggyback_buffer():
    S.step_push_pull_step(100, 64, 40, rounds=12, every=3, pb_cap=2)


def test_no_partner_cases():
    S.no_partner_cases()


def test_same_round_same_partners():
    S.same_round_same_partners(90)


def test_save_push_pull_load():
    S.save_push_pull_load(160)


@pytest.mark.parametrize("cap", [32, 64])
def test_inserts_then_rounds(cap):
    S.inserts_then_rounds(200, cap, deg=cap // 3, rounds=50)


def test_hub():
    S.inserts_then_rounds(300, 32, deg=3, rounds=20, kind="ring", seed=13)


def test_full_rows_drop_inserts():
    S.full_rows_drop_inserts()


def test_push_pull_then_edits():
    S.push_pull_then_edits(160)


def test_export_after_push_pull():
    S.export_after_push_pull(80)


def test_error_paths():
    S.error_paths()
