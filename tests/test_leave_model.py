"""The C oracle's graceful leaves (oracle_leave in tests/between_steps_oracle.c) against the independent restatement in
tests/between_steps_model.py (leave, over oracle/core_model.py's name-keyed stores) on random views and lists: the
oracle's state is copied into model stores, both run the same id list, and every view entry, incarnation, piggyback
buffer, the process arrays, the outputs and the counters must agree, under both protocol flags and the Lifeguard
timeout."""
import numpy as np
import pytest

from between_steps_model import assert_same_state, leave, name, setup, to_model, up_of, variant
from between_steps_oracle import leave as oracle_leave
from swim_b200 import _abi as A


def compare(orc, cfg, ids):
    """One leave on both; returns the oracle's outputs."""
    stores = to_model(orc, cfg)
    alive, back, crash = (orc.get_array(a).copy() for a in (A.ARR_ALIVE, A.ARR_BACK_AT, A.ARR_LAST_CRASH))
    c0 = orc.counters()
    want = leave(stores, up_of(orc), [name(int(i)) for i in ids], cfg.pb_cap, cfg.retransmit, **variant(cfg))
    got = oracle_leave(orc, ids)
    dc = orc.counters() - c0
    assert got == (len(want["left"]), want["delivered"])
    assert (dc[A.CTR_RECS_APPLIED], dc[A.CTR_PB_DROPPED], dc[A.CTR_REFUTES]) == (want["applied"], want["dropped"], 0)
    gone = np.array([int(k) for k in want["left"]], np.int64)
    alive[gone], back[gone], crash[gone] = 0, 0, orc.round
    assert np.array_equal(orc.get_array(A.ARR_ALIVE), alive)
    assert np.array_equal(orc.get_array(A.ARR_BACK_AT), back)
    assert np.array_equal(orc.get_array(A.ARR_LAST_CRASH), crash)
    assert_same_state(orc, stores, cfg)
    return got


def test_leavers_that_list_each_other():
    orc, cfg = setup(16, "ring", 4, rounds=2)
    assert compare(orc, cfg, [3, 4, 5]) == (3, 6)  # ring of degree 4: 1, 2, 6, 7 hear from two leavers or one


def test_repeated_and_down_ids():
    orc, cfg = setup(20, "random", 6, rounds=3, crashes=(2, 7))
    got = compare(orc, cfg, [2, 7, 9, 9, 9, 11, 2])
    assert got[0] == 2


def test_hub_recipient_drops_records():
    n = 200
    orc, cfg = setup(n, "complete", 32, cap=256, rounds=1)
    got = compare(orc, cfg, np.arange(1, 60))
    assert got[0] == 59


@pytest.mark.parametrize("flags,suspicion_max", [(0, 0), (A.F_STRICT_OVERRIDE, 0), (0, 9), (A.F_STRICT_OVERRIDE, 9)])
@pytest.mark.parametrize("kind", ["random", "symmetric"])
def test_random_views_and_lists(flags, suspicion_max, kind):
    orc, cfg = setup(24, kind, 6, seed=9, rounds=5, crashes=(4, 11), loss_ppm=150000, flags=flags,
                     suspicion_max=suspicion_max)
    rng = np.random.default_rng(9 + flags + suspicion_max)
    for _ in range(3):
        compare(orc, cfg, rng.integers(0, 24, size=5))
        orc.step(3)


def test_errors_change_nothing():
    from oracle.oracle import OracleError
    orc, cfg = setup(8, "ring", 2)
    before = orc.get_array(A.ARR_ALIVE).copy()
    for ids in ([8], [1, 9]):
        with pytest.raises(OracleError):
            oracle_leave(orc, ids)
    assert np.array_equal(orc.get_array(A.ARR_ALIVE), before)
    assert oracle_leave(orc, []) == (0, 0)
