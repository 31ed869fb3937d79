"""The C oracle's push-pull exchange (tests/push_pull_oracle.c) against the independent restatement in
tests/push_pull_model.py (over oracle/core_model.py's name-keyed stores, with the reference's own guard order) on small
graphs: the oracle's state is copied into model stores, both run the exchange, and every view entry, incarnation,
piggyback buffer, output and counter must agree, under both protocol flags and the Lifeguard timeout."""
import numpy as np
import pytest

from oracle import core_model as M
from oracle.oracle import Oracle, philox
from push_pull_model import push_pull as model_push_pull
from push_pull_oracle import push_pull as oracle_push_pull
from swim_b200 import _abi as A
from swim_b200.sim import crash_events, default_config, generate_topology

NM = A.NO_MEMBER
KIND = {A.MSG_ALIVE: "Alive", A.MSG_SUSPECT: "Suspect", A.MSG_DEAD: "Dead"}


def name(i):
    return f"{i:05d}"  # key order == id order


def lifeguard_deltas(cfg):
    """What the c-th confirmation takes off a countdown: timeout(c) = max - (max - min) log(c + 1) / log 4, c = 0..3, in
    256ths rounded (the oracle's table)."""
    if not cfg.suspicion_max:
        return None
    frac = (0, 128, 203, 256)
    T = [cfg.suspicion_max - ((cfg.suspicion_max - cfg.suspicion_rounds) * f + 128) // 256 for f in frac]
    return [0] + [T[c - 1] - T[c] for c in range(1, 4)]


def to_model(orc, cfg):
    n, cap = cfg.n_nodes, cfg.view_cap
    lg = cfg.suspicion_max != 0
    nb, st, inc, last = (orc.get_array(a).reshape(n, cap) for a in (A.ARR_NBR, A.ARR_VST, A.ARR_VINC, A.ARR_VLAST))
    pb, cnt = orc.get_array(A.ARR_PB).reshape(n, cfg.pb_cap), orc.get_array(A.ARR_PB_CNT)
    stores = {}
    for i in range(n):
        s = M.Store(M.Member(name(i)), cfg.suspicion_max or cfg.suspicion_rounds)
        s.conf = {}
        s.incarnation = int(orc.get_array(A.ARR_SELF_INC)[i])
        s.now = orc.round
        for x in range(cap):
            if st[i, x] & 3 == A.VACANT:
                continue
            m = name(int(nb[i, x]))
            s.members[m] = M.Member(m, "", 0, 0, int(st[i, x] & 3), int(inc[i, x]), int(last[i, x]))
            if st[i, x] & 3 == A.SUSPECT:
                s.timers[m] = (int(st[i, x]) >> 2) & (15 if lg else 63)
                if lg and st[i, x] >> 6:
                    s.conf[m] = int(st[i, x]) >> 6
        s.queue = [(M.Msg(KIND[int(r["kind"])], node=name(int(r["member"])), incarnation=int(r["incarnation"]),
                          dead_from=name(int(r["from"])) if r["kind"] == A.MSG_DEAD else ""), int(r["ttl"]))
                   for r in pb[i, : cnt[i]]]
        stores[name(i)] = s
    return stores


def model_arrays(stores, cfg):
    n, cap = cfg.n_nodes, cfg.view_cap
    nb = np.full((n, cap), NM, np.uint32)
    st = np.full((n, cap), A.VACANT, np.uint8)
    inc = np.zeros((n, cap), np.uint32)
    last = np.zeros((n, cap), np.uint32)
    pb = []
    for i in range(n):
        s = stores[name(i)]
        for x, m in enumerate(M.members(s)):
            nb[i, x], inc[i, x], last[i, x] = int(m.name), m.incarnation, m.last_change
            if m.alive == A.SUSPECT:
                st[i, x] = m.alive | (s.timers.get(m.name, 0) << 2) | (s.conf.get(m.name, 0) << 6)
            else:
                st[i, x] = m.alive
        pb.append([(int(m.node), {"Alive": A.MSG_ALIVE, "Suspect": A.MSG_SUSPECT, "Dead": A.MSG_DEAD}[m.kind],
                    m.incarnation, int(m.dead_from) if m.kind == "Dead" else 0, t) for m, t in s.queue])
    self_inc = np.array([stores[name(i)].incarnation for i in range(n)], np.uint32)
    return nb, st, inc, last, self_inc, pb


def oracle_pb(orc, cfg):
    pb, cnt = orc.get_array(A.ARR_PB).reshape(cfg.n_nodes, cfg.pb_cap), orc.get_array(A.ARR_PB_CNT)
    return [[(int(r["member"]), int(r["kind"]), int(r["incarnation"]), int(r["from"]), int(r["ttl"])) for r in pb[i, : cnt[i]]]
            for i in range(cfg.n_nodes)]


def compare(orc, cfg):
    """One exchange on both; returns the oracle's outputs."""
    stores = to_model(orc, cfg)
    up = {name(i): bool(a) for i, a in enumerate(orc.get_array(A.ARR_ALIVE))}
    key = (cfg.seed & 0xFFFFFFFF, cfg.seed >> 32)
    r = orc.round
    draw = lambda k: philox([r, int(k), 10, 0], key)[0]
    c0 = orc.counters()
    want = model_push_pull(stores, up, draw, cfg.view_cap, cfg.pb_cap, cfg.retransmit,
                           strict=bool(cfg.flags & A.F_STRICT_OVERRIDE), lg_delta=lifeguard_deltas(cfg))
    got = oracle_push_pull(orc)
    dc = orc.counters() - c0
    assert got == (want["exchanges"], want["inserted"], want["full"])
    assert (dc[A.CTR_RECS_APPLIED], dc[A.CTR_REFUTES], dc[A.CTR_PB_DROPPED]) == (want["applied"], want["refutes"], want["dropped"])
    nb, st, inc, last, self_inc, pb = model_arrays(stores, cfg)
    n, cap = cfg.n_nodes, cfg.view_cap
    assert np.array_equal(orc.get_array(A.ARR_NBR).reshape(n, cap), nb)
    assert np.array_equal(orc.get_array(A.ARR_VST).reshape(n, cap), st)
    assert np.array_equal(orc.get_array(A.ARR_VINC).reshape(n, cap), inc)
    assert np.array_equal(orc.get_array(A.ARR_VLAST).reshape(n, cap), last)
    assert np.array_equal(orc.get_array(A.ARR_SELF_INC), self_inc)
    assert oracle_pb(orc, cfg) == pb
    return got


def setup(n, kind, deg, seed=1, rounds=0, crashes=(), cap=32, **kw):
    cfg = default_config(n_nodes=n, view_cap=cap, seed=seed, suspicion_rounds=4, **kw)
    orc = Oracle(cfg)
    orc.set_view(generate_topology(kind, n, cap, deg, seed=seed))
    if crashes:
        orc.inject(crash_events(1, list(crashes)))
    if rounds:
        orc.step(rounds)
    return orc, cfg


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
