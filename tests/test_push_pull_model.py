"""The C oracle's push-pull exchange (tests/between_steps_oracle.c) against the independent restatement in
tests/between_steps_model.py (over oracle/core_model.py's name-keyed stores, with the reference's own guard order) on
small graphs: the oracle's state is copied into model stores, both run the exchange, and every view entry, incarnation,
piggyback buffer, output and counter must agree, under both protocol flags and the Lifeguard timeout."""
import numpy as np
import pytest

from between_steps_model import assert_same_state, push_pull, setup, to_model, up_of, variant
from between_steps_oracle import push_pull as oracle_push_pull
from oracle.oracle import Oracle, philox
from swim_b200 import _abi as A
from swim_b200.sim import default_config

NM = A.NO_MEMBER


def compare(orc, cfg):
    """One exchange on both; returns the oracle's outputs."""
    stores = to_model(orc, cfg)
    key = (cfg.seed & 0xFFFFFFFF, cfg.seed >> 32)
    r = orc.round
    draw = lambda k: philox([r, int(k), 10, 0], key)[0]
    c0 = orc.counters()
    want = push_pull(stores, up_of(orc), draw, cfg.view_cap, cfg.pb_cap, cfg.retransmit, **variant(cfg))
    got = oracle_push_pull(orc)
    dc = orc.counters() - c0
    assert got == (want["exchanges"], want["inserted"], want["full"])
    assert (dc[A.CTR_RECS_APPLIED], dc[A.CTR_REFUTES], dc[A.CTR_PB_DROPPED]) == (want["applied"], want["refutes"], want["dropped"])
    assert_same_state(orc, stores, cfg)
    return got


@pytest.mark.parametrize("kind,deg,n", [("complete", 32, 12), ("ring", 2, 16), ("ring", 6, 16), ("random", 5, 16)])
def test_views(kind, deg, n):
    orc, cfg = setup(n, kind, deg, rounds=3, loss_ppm=100000)
    got = compare(orc, cfg)
    assert got[0] > 0
    if kind != "complete":
        assert got[1] > 0  # D < cap: unknown members are inserted
    for _ in range(3):  # later rounds: other partners, states that have moved on
        orc.step(2)
        compare(orc, cfg)


def test_full_row_drops_inserts():
    orc, cfg = setup(40, "random", 32, seed=2)
    got = compare(orc, cfg)
    assert got[2] > 0 and got[1] == 0


def test_hub():
    """Node 0 is listed by everybody else and holds no Alive member: all choosers of a ring cross at one receiver."""
    n, cap = 16, 32
    cfg = default_config(n_nodes=n, view_cap=cap, seed=3, suspicion_rounds=4)
    nbr = np.full((n, cap), NM, np.uint32)
    for i in range(1, n):
        nbr[i, 0] = 0
    nbr[0, 0] = 1
    orc = Oracle(cfg)
    orc.set_view(nbr)
    got = compare(orc, cfg)
    assert got[0] == n and got[1] > 0


def test_mutual_partners():
    """Two nodes listing only each other pick each other: each sends once and receives once."""
    n, cap = 2, 32
    cfg = default_config(n_nodes=n, view_cap=cap, seed=4)
    nbr = np.full((n, cap), NM, np.uint32)
    nbr[0, 0], nbr[1, 0] = 1, 0
    orc = Oracle(cfg)
    orc.set_view(nbr)
    assert compare(orc, cfg) == (2, 0, 0)


def test_crashed_partner_and_no_alive_slot():
    orc, cfg = setup(16, "ring", 2, rounds=12, crashes=(3, 4, 5, 9))
    compare(orc, cfg)
    orc, cfg = setup(6, "complete", 32, crashes=range(6), rounds=2)
    assert compare(orc, cfg) == (0, 0, 0)


def test_refutation_of_a_suspect_or_dead_receiver():
    """Node 1 is Suspect in some rows and Dead in others; when those rows reach it, it refutes."""
    orc, cfg = setup(12, "complete", 32, seed=5)
    st = orc.get_array(A.ARR_VST).reshape(12, 32)
    st[2:12, 0] = A.SUSPECT | (4 << 2)
    st[6:12, 0] = A.DEAD
    orc.set_array(A.ARR_VST, st.reshape(-1))
    c0 = orc.counters()
    compare(orc, cfg)
    assert (orc.counters() - c0)[A.CTR_REFUTES] > 0


@pytest.mark.parametrize("flags,suspicion_max", [(0, 0), (A.F_STRICT_OVERRIDE, 0), (0, 9), (A.F_STRICT_OVERRIDE, 9)])
def test_suspect_about_a_suspect(flags, suspicion_max):
    """Rows that already suspect a member receive Suspect about it from partners: a `Nothing` for the reference, a
    Lifeguard confirmation with suspicion_max; Dead about it replaces it in other rows, and under STRICT_OVERRIDE a
    Suspect of a newer incarnation overrides the older suspicion."""
    orc, cfg = setup(10, "complete", 32, seed=6, flags=flags, suspicion_max=suspicion_max)
    st = orc.get_array(A.ARR_VST).reshape(10, 32)
    inc = orc.get_array(A.ARR_VINC).reshape(10, 32)
    st[:, 4] = A.SUSPECT | (3 << 2)
    st[5:, 4] = A.DEAD
    st[:, 7] = A.SUSPECT | (4 << 2)
    inc[:4, 7] = 2  # rows 0..3 hold a newer suspicion of the member in slot 7 than the others
    orc.set_array(A.ARR_VST, st.reshape(-1))
    orc.set_array(A.ARR_VINC, inc.reshape(-1))
    assert compare(orc, cfg)[0] == 10
    if suspicion_max:
        assert (orc.get_array(A.ARR_VST) >> 6).any()  # some countdowns were confirmed


@pytest.mark.parametrize("flags,suspicion_max", [(A.F_STRICT_OVERRIDE, 0), (0, 9)])
def test_variants_after_rounds(flags, suspicion_max):
    orc, cfg = setup(16, "random", 6, seed=9, rounds=5, crashes=(4, 11), loss_ppm=150000, flags=flags,
                     suspicion_max=suspicion_max)
    for _ in range(3):
        compare(orc, cfg)
        orc.step(2)


def test_piggyback_overflow():
    orc, cfg = setup(16, "ring", 4, seed=7, rounds=6, pb_cap=2, crashes=(2, 9))
    c0 = orc.counters()
    compare(orc, cfg)
    assert (orc.counters() - c0)[A.CTR_PB_DROPPED] > 0


def test_same_round_same_partners():
    orc, cfg = setup(16, "complete", 32, seed=8)
    a = compare(orc, cfg)
    assert compare(orc, cfg)[0] == a[0]
