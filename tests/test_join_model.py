"""The C oracle's seed joins (oracle_join in tests/between_steps_oracle.c) against the independent restatement in
tests/between_steps_model.py (join, over oracle/core_model.py's name-keyed stores) on small graphs: the oracle's state
is copied into model stores, both run the same pair list, and every view entry, incarnation, piggyback buffer, output
and counter must agree, under both protocol flags and the Lifeguard timeout."""
import numpy as np
import pytest

from between_steps_model import assert_same_state, join, name, setup, to_model, up_of, variant
from between_steps_oracle import join as oracle_join
from swim_b200 import _abi as A


def compare(orc, cfg, nodes, seeds, fresh=False):
    """One join on both; returns the oracle's outputs."""
    stores = to_model(orc, cfg)
    c0 = orc.counters()
    want = join(stores, up_of(orc), [(name(j), name(s)) for j, s in zip(nodes, seeds)], cfg.view_cap, cfg.pb_cap,
                cfg.retransmit, fresh, **variant(cfg))
    got = oracle_join(orc, nodes, seeds, fresh)
    dc = orc.counters() - c0
    assert got == (want["exchanges"], want["inserted"], want["full"])
    assert (dc[A.CTR_RECS_APPLIED], dc[A.CTR_REFUTES], dc[A.CTR_PB_DROPPED]) == (want["applied"], want["refutes"], want["dropped"])
    assert_same_state(orc, stores, cfg)
    return got


def test_empty_joiner_rows():
    orc, cfg = setup(16, "ring", 4, rounds=2)
    assert compare(orc, cfg, [3, 9], [12, 1], fresh=True)[1] > 0
    orc.step(2)
    assert compare(orc, cfg, [3, 4], [4, 3], fresh=True) == (2, 2, 0)  # both rows empty: Alive(self) only


def test_joiner_does_not_list_its_seed():
    orc, cfg = setup(20, "ring", 2, rounds=1)
    assert 10 not in orc.get_array(A.ARR_NBR).reshape(20, 32)[0]
    assert compare(orc, cfg, [0], [10])[1] > 0


def test_mutual_and_duplicated_pairs():
    orc, cfg = setup(16, "random", 5, rounds=3, loss_ppm=100000)
    got = compare(orc, cfg, [1, 1, 2, 5, 6], [2, 2, 1, 6, 5])
    assert got[0] == 5


def test_hub_seed_with_thousands_of_joiners():
    n = 3000
    orc, cfg = setup(n, "ring", 4, rounds=1)
    others = np.arange(1, n)
    got = compare(orc, cfg, others, np.zeros(n - 1, np.int64), fresh=True)
    assert got[0] == n - 1 and got[2] > 0


def test_down_seed_and_down_joiner():
    orc, cfg = setup(16, "ring", 4, rounds=3, crashes=(2, 7))
    assert compare(orc, cfg, [2, 3, 7, 8], [5, 7, 9, 9], fresh=True)[0] == 1


def test_full_rows():
    orc, cfg = setup(40, "random", 32, seed=2)
    got = compare(orc, cfg, [0, 1, 2], [20, 21, 22])
    assert got[2] > 0 and got[1] == 0


def test_refutation_at_a_suspect_or_dead_receiver():
    """Node 0 is Suspect in rows 2..5 and Dead in rows 6..11; joining through three of them, it refutes."""
    orc, cfg = setup(12, "complete", 32, seed=5)
    st = orc.get_array(A.ARR_VST).reshape(12, 32)
    st[2:12, 0] = A.SUSPECT | (4 << 2)
    st[6:12, 0] = A.DEAD
    orc.set_array(A.ARR_VST, st.reshape(-1))
    c0 = orc.counters()
    compare(orc, cfg, [0, 0, 0], [3, 7, 9])  # rows 2.. list node 0 in slot 0
    assert (orc.counters() - c0)[A.CTR_REFUTES] > 0


@pytest.mark.parametrize("flags,suspicion_max", [(0, 0), (A.F_STRICT_OVERRIDE, 0), (0, 9), (A.F_STRICT_OVERRIDE, 9)])
@pytest.mark.parametrize("fresh", [False, True])
def test_variants_after_rounds(flags, suspicion_max, fresh):
    orc, cfg = setup(16, "random", 6, seed=9, rounds=5, crashes=(4, 11), loss_ppm=150000, flags=flags,
                     suspicion_max=suspicion_max)
    rng = np.random.default_rng(9)
    for _ in range(3):
        nodes = rng.integers(0, 16, size=8)
        seeds = (nodes + rng.integers(1, 16, size=8)) % 16
        compare(orc, cfg, nodes, seeds, fresh)
        orc.step(2)


def test_errors_change_nothing():
    from oracle.oracle import OracleError
    orc, cfg = setup(8, "ring", 2)
    before = orc.get_array(A.ARR_NBR).copy()
    for nodes, seeds in (([1], [1]), ([8], [1]), ([1], [9])):
        with pytest.raises(OracleError):
            oracle_join(orc, nodes, seeds, True)
    assert np.array_equal(orc.get_array(A.ARR_NBR), before)
    assert oracle_join(orc, [], []) == (0, 0, 0)
