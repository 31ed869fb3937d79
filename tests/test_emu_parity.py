"""The device code on the CPU. tests/emu compiles the library's own CUDA sources (swim_b200/csrc/*.cu, swim_device.cuh)
with g++ against a SIMT emulator (a warp = one OS thread, a lane = one fiber; see tests/emu/include/cuda_runtime.h) into
tests/emu/libswim_emu.so, which exports the same C ABI. These tests point the ctypes loader at it — a test-only switch —
and repeat the parity scenarios of the `-m gpu` suite at small sizes against the oracle: the same kernels (grid barriers,
warp ballots, candidate slots, claim stamps, peer-memory exchange with several ranks in one process) without a GPU.
What the emulator cannot show: real memory-model effects, occupancy, performance."""
import ctypes as C
import threading

import numpy as np
import pytest

from helpers import assert_same_state, concat_events, crash_events, default_config, generate_topology, make_pair, random_events
from spec_fixture import member, msg
from swim_b200 import _abi as A


@pytest.fixture(scope="module", autouse=True)
def emu_library():
    import os
    import sys
    import swim_b200._lib as L
    here = os.path.dirname(os.path.abspath(__file__))
    sys.path.insert(0, os.path.join(here, "emu"))
    import build_emu
    so = build_emu.build()
    saved = (L.SO_PATH, L._lib)
    L.SO_PATH, L._lib = so, None
    assert L.lib().swim_abi_version() == A.ABI_VERSION
    yield
    L.SO_PATH, L._lib = saved


def test_c1_every_round():
    cfg = default_config(n_nodes=32, seed=0x5EED0001 + 1)
    nbr = generate_topology("complete", 32, 32)
    sim, orc = make_pair(cfg, nbr)
    ev = crash_events(10, [7, 19])
    sim.inject(ev)
    orc.inject(ev)
    for r in range(100):
        sim.step(1)
        orc.step(1)
        assert_same_state(sim, orc, f"round {r + 1}")
    assert sim.mismatches() == 0


@pytest.mark.parametrize("flags", [0, A.F_STRICT_OVERRIDE, A.F_ROUND_ROBIN, A.F_STRICT_OVERRIDE | A.F_ROUND_ROBIN])
@pytest.mark.parametrize("seed", range(3))
def test_random_small(seed, flags):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(2, 160))
    deg = int(rng.integers(1, min(n - 1, 32) + 1))
    k = int(rng.integers(0, 8))
    cfg = default_config(n_nodes=n, view_cap=32, k_indirect=k, fanout=int(rng.integers(1, k + 2)),
                         pb_cap=int(rng.integers(1, 33)), suspicion_rounds=int(rng.integers(1, 12)),
                         retransmit=int(rng.integers(1, 12)), loss_ppm=int(rng.choice([0, 0, 50000, 300000])),
                         seed=int(rng.integers(0, 2 ** 63)), flags=flags)
    kind = rng.choice(["random", "ring"]) if deg < n - 1 else "complete"
    nbr = generate_topology(str(kind), n, 32, deg, seed=seed + 1)
    sim, orc = make_pair(cfg, nbr)
    rounds = 70 if flags & A.F_ROUND_ROBIN else 40
    ev = random_events(rng, n, rounds, n_crash=max(1, n // 10), n_rejoin=max(1, n // 30), n_inject=n // 4)
    sim.inject(ev)
    orc.inject(ev)
    for r in range(rounds):
        sim.step(1)
        orc.step(1)
        assert_same_state(sim, orc, f"flags {flags} seed {seed} round {r + 1}")


@pytest.mark.parametrize("cap,flags", [(64, 0), (128, A.F_ROUND_ROBIN), (256, A.F_STRICT_OVERRIDE | A.F_ROUND_ROBIN)])
def test_wide_rows(cap, flags):
    rng = np.random.default_rng(cap)
    n = 120
    cfg = default_config(n_nodes=n, view_cap=cap, k_indirect=5, fanout=4, pb_cap=16, suspicion_rounds=3, retransmit=5,
                         loss_ppm=20000, seed=cap, flags=flags)
    nbr = generate_topology("random", n, cap, min(cap - 7, n - 1), seed=3)
    sim, orc = make_pair(cfg, nbr)
    ev = random_events(rng, n, 30, n_crash=12, n_rejoin=5, n_inject=20)
    sim.inject(ev)
    orc.inject(ev)
    for r in range(30):
        sim.step(1)
        orc.step(1)
        assert_same_state(sim, orc, f"cap {cap} round {r + 1}")


def test_multi_round_launches_equal_single_steps():
    """round_kernel runs every event-free stretch of a call in one launch (grid barriers inside)."""
    rng = np.random.default_rng(9)
    n = 300
    cfg = default_config(n_nodes=n, seed=77)
    nbr = generate_topology("random", n, 32, 20, seed=2)
    ev = random_events(rng, n, 60, n_crash=20, n_rejoin=6, n_inject=10)
    a, orc = make_pair(cfg, nbr)
    a.inject(ev)
    orc.inject(ev)
    for chunk in (1, 7, 2, 30, 20):
        a.step(chunk)
        orc.step(chunk)
        assert_same_state(a, orc, f"after a chunk of {chunk}")


def test_scalar_calls_match_oracle():
    from oracle.oracle import Oracle, OracleError
    from swim_b200._lib import check, lib
    from swim_b200.sim import Simulator
    rng = np.random.default_rng(11)
    for flags in (0, A.F_STRICT_OVERRIDE):
        cfg = default_config(n_nodes=256, view_cap=32, suspicion_rounds=7, flags=flags)
        sim, orc = Simulator(cfg), Oracle(cfg)
        node = 100
        ms = [member(int(i), int(rng.integers(0, 3)), int(rng.integers(0, 4))) for i in rng.choice(90, 20, replace=False)]
        for m in ms:
            m.timer = 3 if m.liveness == A.SUSPECT else 0
        check(lib().swim_set_members(sim._h, node, (A.Member * len(ms))(*ms), len(ms)), "set", sim._h)
        orc.set_members(node, ms)
        fns = {A.MSG_SUSPECT: (lib().swim_suspect_node, orc.suspect_node), A.MSG_DEAD: (lib().swim_dead_node, orc.dead_node),
               A.MSG_ALIVE: (lib().swim_alive_node, orc.alive_node)}
        for step in range(150):
            kind = int(rng.choice([A.MSG_SUSPECT, A.MSG_DEAD, A.MSG_ALIVE]))
            who = int(rng.choice([node, int(rng.integers(0, 90)), int(rng.integers(0, 90))]))
            if who == node and kind == A.MSG_ALIVE:
                who = int(rng.integers(0, 90))
            m = msg(kind, who, int(rng.integers(0, 6)), dead_from=int(rng.integers(0, 90)))
            out, has = A.Message(), C.c_int()
            rc = fns[kind][0](sim._h, node, C.byref(m), C.byref(out), C.byref(has))
            try:
                exp = fns[kind][1](node, m)
            except OracleError as e:
                assert (rc, e.code) == (A.ECAP, A.ECAP)
                continue
            assert rc == 0 and bool(has.value) == (exp is not None), (flags, step, kind, who)
            if exp is not None:
                assert (out.kind, out.node, out.incarnation, out.dead_from) == (exp.kind, exp.node, exp.incarnation, exp.dead_from)
            buf, cnt = (A.Member * 32)(), C.c_size_t()
            check(lib().swim_get_members(sim._h, node, buf, 32, C.byref(cnt)), "get", sim._h)
            got = [(buf[i].id, buf[i].liveness, buf[i].timer, buf[i].incarnation) for i in range(cnt.value)]
            assert got == [(x.id, x.liveness, x.timer, x.incarnation) for x in orc.get_members(node)], step
            if step % 7 == 3:  # the per-period steps of a real-time node: countdown, piggyback payload
                e = C.c_uint32()
                check(lib().swim_tick_timers(sim._h, node, C.byref(e)), "tick", sim._h)
                assert e.value == orc.tick_timers(node), step
                mb, mc = (A.Message * A.MAX_PB)(), C.c_size_t()
                check(lib().swim_take_broadcasts(sim._h, node, mb, A.MAX_PB, C.byref(mc)), "take", sim._h)
                assert [(mb[i].kind, mb[i].node, mb[i].incarnation, mb[i].dead_from) for i in range(mc.value)] == \
                    [(x.kind, x.node, x.incarnation, x.dead_from) for x in orc.take_broadcasts(node)], step
            elif exp is not None:
                check(lib().swim_broadcast(sim._h, node, C.byref(out)), "bc", sim._h)
                orc.broadcast(node, exp)
        for n_pick in (0, 1, 5, 64):
            buf, cnt = (A.Member * 32)(), C.c_size_t()
            check(lib().swim_k_random_members(sim._h, node, n_pick, None, 0, buf, 32, C.byref(cnt)), "krm", sim._h)
            assert [buf[i].id for i in range(cnt.value)] == [x.id for x in orc.k_random_members(node, n_pick, [])]
        sim.step(3)
        orc.step(3)
        assert sim.digest() == orc.digest()


# ---------------------------------------------------------------- several ranks in one process (fused exchange)
from helpers import run_sharded  # noqa: E402


@pytest.mark.parametrize("path", ["split", "round_kernel"])
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_fused_exchange_equals_oracle(world, path, monkeypatch):
    """round_kernel (the default for shards): one launch per event-free stretch, the last CTA of a grid barrier does the
    cross-GPU handshake; split (SWIM_ROUND_KERNEL=0): K1a / K1b / peer_barrier_kernel / K2 as separate launches."""
    monkeypatch.setenv("SWIM_ROUND_KERNEL", "1" if path == "round_kernel" else "0")
    run_sharded(world, n=403, chunks=[1] * 6 + [12], loss=20000, deg=24)


def test_sharded_variants(monkeypatch):
    monkeypatch.setenv("SWIM_ROUND_KERNEL", "1")
    run_sharded(2, n=200, chunks=[1, 1, 40], loss=0, deg=20, flags=A.F_STRICT_OVERRIDE | A.F_ROUND_ROBIN)


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_staged_exchange_equals_oracle(world, monkeypatch):
    """The NCCL baseline path (bucketed envelopes, all-gathered counts, send/recv per peer, deliver_kernel) with an in-process
    stand-in for the nine NCCL calls the library binds at run time."""
    import os
    here = os.path.dirname(os.path.abspath(__file__))
    monkeypatch.setenv("SWIM_NCCL_LIB", os.path.join(here, "emu", "libfake_nccl.so"))
    run_sharded(world, n=403, chunks=[1] * 5 + [9], loss=20000, deg=24, mode="nccl")


def test_checkpoint_and_resume():
    """State arrays + round counter reproduce a run exactly: a fresh handle restored from a checkpoint continues with the
    same digests as the run it was taken from (and as the oracle)."""
    from swim_b200.sim import Simulator
    rng = np.random.default_rng(5)
    n = 240
    cfg = default_config(n_nodes=n, seed=31, loss_ppm=30000)
    nbr = generate_topology("random", n, 32, 20, seed=8)
    ev = random_events(rng, n, 60, n_crash=20, n_rejoin=6, n_inject=30)
    a, orc = make_pair(cfg, nbr)
    a.inject(ev)
    orc.inject(ev)
    a.step(25)
    orc.step(25)
    ck = a.checkpoint()
    assert ck["round"] == 25
    b = Simulator(default_config(n_nodes=n, seed=31, loss_ppm=30000))
    b.restore(ck)
    b.inject(ev[ev["round"] > 25])
    assert b.round == 25 and b.digest() == a.digest()
    for _ in range(7):
        a.step(5)
        b.step(5)
        orc.step(5)
        assert a.digest() == b.digest() == orc.digest()
    assert np.array_equal(a.get_array(A.ARR_VLAST), b.get_array(A.ARR_VLAST))
    # counters are cumulative since create: the resumed handle counts from the checkpoint on
    assert (a.counters() - b.counters()).min() >= 0


@pytest.mark.parametrize("loss,flags", [(0, 0), (1500, 0), (700, A.F_ROUND_ROBIN), (6000, A.F_STRICT_OVERRIDE)])
def test_long_launches_through_quiet_and_busy_stretches(loss, flags):
    """One call = one launch per event-free stretch. Quiescent stretches (a healthy cluster) and rounds with work alternate:
    rarely lost probes raise a suspicion now and then, a crash lands in the middle. State AND counters (every Ping is
    counted exactly once) must equal the oracle's wherever the kernel stops batching rounds."""
    n = 300
    cfg = default_config(n_nodes=n, seed=1234 + loss, loss_ppm=loss, flags=flags)
    nbr = generate_topology("random", n, 32, 24, seed=5)
    sim, orc = make_pair(cfg, nbr)
    ev = crash_events(57, [17, 200])
    sim.inject(ev)
    orc.inject(ev)
    for chunk in (3, 41, 100, 7, 120):
        sim.step(chunk)
        orc.step(chunk)
        assert_same_state(sim, orc, f"loss {loss} after {sim.round} rounds")
    import os
    if not any(os.environ.get(k) for k in ("SWIM_SPLIT", "SWIM_ONE_ROUND_PER_LAUNCH")):
        assert sim.launch_count() < 40  # one launch per event-free stretch (+ digests of the comparisons)


@pytest.mark.parametrize("qbatch,flags,cap", [("0", 0, 32), ("2", 0, 32), ("5", A.F_ROUND_ROBIN, 32), ("8", 0, 32),
                                              ("8", A.F_STRICT_OVERRIDE, 32), ("4", 0, 64), ("7", A.F_ROUND_ROBIN, 128)])
def test_batched_quiet_scans(qbatch, flags, cap, monkeypatch):
    """round_kernel decides up to SWIM_QUIET_BATCH rounds per pass once a round listed no work (quiet_scan). Two crashed
    nodes sit in 32 views each: for a long while a round is busy only when some observer's draw hits one of them, so quiet
    and busy rounds alternate inside a launch and batches end early at every position; later the cluster is converged and
    whole batches commit, including the short one at the end of a launch. State and counters equal the oracle's."""
    monkeypatch.setenv("SWIM_QUIET_BATCH", qbatch)
    n = 230
    cfg = default_config(n_nodes=n, view_cap=cap, seed=99 + int(qbatch), suspicion_rounds=2, retransmit=2, flags=flags)
    nbr = generate_topology("random", n, cap, cap - 7 if cap > 32 else 32, seed=11)
    sim, orc = make_pair(cfg, nbr)
    ev = concat_events([crash_events(4, [101]), crash_events(90, [7])])
    sim.inject(ev)
    orc.inject(ev)
    for chunk in (1, 2, 3, 61, 9, 40, 2, 130, 64, 11):
        sim.step(chunk)
        orc.step(chunk)
        assert_same_state(sim, orc, f"qbatch {qbatch} after {sim.round} rounds")


@pytest.mark.parametrize("kind,deg,cap", [("random", 6, 32), ("ring", 12, 32), ("random", 40, 64)])
def test_sender_side_membership_filter(kind, deg, cap):
    """K1b tests every envelope against the recipient's membership filter (256 W bits per node) and delivers only those
    that can matter. Sparse random views: nearly every envelope is dropped at its sender (receivers do not know the
    member), K2 is skipped in most rounds; ring views: nearly everything is delivered. Either way every array, the
    counters (envelopes received by live processes are counted at the sender) and the digest equal the oracle's."""
    rng = np.random.default_rng(deg)
    n = 3000 if kind == "random" else 600
    cfg = default_config(n_nodes=n, view_cap=cap, seed=1234 + deg, suspicion_rounds=3, pb_cap=6, retransmit=5)
    nbr = generate_topology(kind, n, cap, deg, seed=deg)
    sim, orc = make_pair(cfg, nbr)
    ev = random_events(rng, n, 40, n_crash=n // 15, n_rejoin=n // 60, n_inject=n // 20)
    sim.inject(ev)
    orc.inject(ev)
    for chunk in (1, 3, 9, 2, 17, 8):
        sim.step(chunk)
        orc.step(chunk)
        assert_same_state(sim, orc, f"{kind} deg {deg} after {sim.round} rounds")
    c = sim.counters()
    assert c[A.CTR_MSGS] > 500 and c[A.CTR_MSGS_RECV] > 0


@pytest.mark.parametrize("flags,ppm", [(0, 20000), (A.F_STRICT_OVERRIDE | A.F_ROUND_ROBIN, 60000)])
def test_device_side_churn_equals_oracle(flags, ppm):
    """BASELINE config C5's churn, generated on the device (churn_kernel -> event_kernel): per-round per-node crash draws
    and rejoin delays from Philox purpose 7, mirrored by the oracle's phase C; mixed with host events on the same nodes."""
    rng = np.random.default_rng(ppm)
    n = 700
    cfg = default_config(n_nodes=n, seed=77, churn_ppm=ppm, rejoin_min=2, rejoin_max=9, suspicion_rounds=3, flags=flags)
    nbr = generate_topology("ring", n, 32, 16, seed=1)
    sim, orc = make_pair(cfg, nbr)
    ev = random_events(rng, n, 40, n_crash=30, n_rejoin=10, n_inject=30)
    sim.inject(ev)
    orc.inject(ev)
    for chunk in (1, 1, 3, 10, 25):
        sim.step(chunk)
        orc.step(chunk)
        assert_same_state(sim, orc, f"churn {ppm} after {sim.round} rounds")
    back = sim.get_array(A.ARR_BACK_AT)
    alive = sim.get_array(A.ARR_ALIVE)
    assert (back > 0).sum() > 0 and (alive == 0).sum() > 0 and sim.counters()[A.CTR_REFUTES] >= 0
    # save / load carry the rejoin schedule
    sim.save()
    d0 = sim.digest()
    sim.step(15)
    orc.step(15)
    assert_same_state(sim, orc, "churn after save + 15")
    sim.load()
    assert sim.digest() == d0
    sim.step(15)
    assert sim.digest() == orc.digest()


def test_device_side_churn_sharded():
    run_sharded(3, n=500, chunks=[1, 2, 9, 20], loss=10000, deg=20, churn=(30000, 2, 7))


def test_many_events_per_round_grouped_by_node():
    """event_kernel gets a round's events grouped by node (stable) and gives each same-node run to one warp: several
    events on one node in one round (crash, rejoin, crash again, injected datagrams) must keep their order, across
    separate swim_sim_inject calls and interleaved with other nodes' events."""
    rng = np.random.default_rng(21)
    n = 200
    cfg = default_config(n_nodes=n, seed=5)
    nbr = generate_topology("random", n, 32, 24, seed=4)
    sim, orc = make_pair(cfg, nbr)
    from swim_b200.sim import make_events
    parts = []
    for r in (2, 3, 5):
        nodes = rng.integers(0, 12, size=60).astype(np.uint32)  # few nodes: long same-node runs
        kinds = rng.choice([A.EV_CRASH, A.EV_REJOIN, A.EV_INJECT], size=60).astype(np.uint8)
        parts.append(make_events(np.full(60, r, np.uint32), nodes, kinds,
                                 msg_kind=rng.choice([A.MSG_SUSPECT, A.MSG_ALIVE, A.MSG_DEAD], size=60).astype(np.uint8),
                                 msg_node=rng.integers(0, n, size=60).astype(np.uint32), msg_inc=rng.integers(0, 3, size=60),
                                 msg_from=rng.integers(0, n, size=60).astype(np.uint32)))
    # two inject calls whose rounds interleave
    a, b = concat_events([parts[0], parts[2]]), parts[1]
    for x in (a, b):
        sim.inject(x)
        orc.inject(x)
    for r in range(12):
        sim.step(1)
        orc.step(1)
        assert_same_state(sim, orc, f"round {r + 1}")


def test_save_load_replays_the_same_rounds():
    """swim_sim_save / swim_sim_load: the device-resident checkpoint brings back state, counters, round and pending events;
    replayed rounds give the same result, also after the handle ran far past the checkpoint (round-stamped scratch arrays
    are cleared), and swim_sim_set_round on a handle that has stepped does the same for the host-side checkpoint."""
    rng = np.random.default_rng(33)
    n = 400
    cfg = default_config(n_nodes=n, seed=91)
    nbr = generate_topology("random", n, 32, 20, seed=6)
    sim, orc = make_pair(cfg, nbr)
    ev = random_events(rng, n, 60, n_crash=30, n_rejoin=8, n_inject=12)
    sim.inject(ev)
    orc.inject(ev)
    sim.step(25)
    orc.step(25)
    assert_same_state(sim, orc, "round 25")
    sim.save()
    ck = sim.checkpoint()
    sim.step(35)
    orc.step(35)
    assert_same_state(sim, orc, "round 60")
    ref = (sim.digest(), sim.counters().tolist())
    for rep in range(2):
        sim.load()
        assert sim.round == 25
        sim.step(35)
        assert (sim.digest(), sim.counters().tolist()) == ref, f"replay {rep}"
    # the host-side checkpoint on the SAME handle: arrays + round (events after round 25 re-injected by the caller)
    sim.restore(ck)
    sim.inject(ev[ev["round"] > 25])
    sim.step(35)
    assert sim.digest() == ref[0]


@pytest.mark.parametrize("flags", [0, A.F_STRICT_OVERRIDE])
def test_dynamic_suspicion_timeout(flags):
    """cfg.suspicion_max (Lifeguard-style): a suspicion starts with suspicion_max rounds and every further Suspect received
    about the suspected member shortens it (timeout(c) = max - (max - min) log(c+1)/log 4, at most 3 confirmations); the
    state byte carries the confirmation count. Ring views so that suspicions about one member meet at its neighbours."""
    rng = np.random.default_rng(8 + flags)
    n = 400
    cfg = default_config(n_nodes=n, seed=3, suspicion_rounds=3, suspicion_max=12, flags=flags, loss_ppm=30000)
    nbr = generate_topology("ring", n, 32, 16, seed=1)
    sim, orc = make_pair(cfg, nbr)
    ev = random_events(rng, n, 50, n_crash=25, n_rejoin=5, n_inject=60)
    sim.inject(ev)
    orc.inject(ev)
    seen_conf = 0
    for r in range(50):
        sim.step(1)
        orc.step(1)
        assert_same_state(sim, orc, f"flags {flags} round {r + 1}")
        vst = sim.get_array(A.ARR_VST)
        seen_conf = max(seen_conf, int((vst[(vst & 3) == A.SUSPECT] >> 6).max(initial=0)))
    assert seen_conf >= 2  # confirmations did arrive
    # detection is faster than with a fixed suspicion_max and never faster than suspicion_rounds allows
    c = sim.counters()
    assert c[A.CTR_DEAD_TIMEOUT] > 0


@pytest.mark.parametrize("probes,flags,loss", [(2, 0, 0), (4, 0, 40000), (3, A.F_ROUND_ROBIN, 0), (4, A.F_STRICT_OVERRIDE | A.F_ROUND_ROBIN, 30000)])
def test_probes_per_round(probes, flags, loss):
    """cfg.probes_per_round = P: the reference's literal `kRandomMembers store numToGossip []` then `mapM_ probeNode'`
    (Core.hs:239-240; SURVEY Q11) — P targets from ONE shuffle, probed one after the other within the period, each with its
    own proxy draw on the store as the earlier probes left it."""
    rng = np.random.default_rng(probes * 10 + flags)
    n = 300
    cfg = default_config(n_nodes=n, seed=5 + probes, probes_per_round=probes, suspicion_rounds=3, loss_ppm=loss, flags=flags)
    nbr = generate_topology("random", n, 32, 12, seed=2)
    sim, orc = make_pair(cfg, nbr)
    ev = random_events(rng, n, 40, n_crash=40, n_rejoin=8, n_inject=20)
    sim.inject(ev)
    orc.inject(ev)
    for chunk in [1] * 8 + [4, 9, 19]:
        sim.step(chunk)
        orc.step(chunk)
        assert_same_state(sim, orc, f"P {probes} flags {flags} after {sim.round} rounds")
    c = sim.counters()
    assert c[A.CTR_PINGS] > (probes - 0.5) * 0.8 * n * 40 * 0.5 and c[A.CTR_SUSPECT_LOCAL] > 0


def test_parameter_sweep_on_one_handle():
    """The C5 study's flow: ONE handle, swim_sim_save at round 0, then per sweep point swim_sim_load +
    swim_sim_set_params (suspicion timeout, Lifeguard start value, churn rate) — each point equals a fresh oracle run with
    that configuration; fields that size the handle are refused."""
    from oracle.oracle import Oracle
    from swim_b200._lib import SwimError
    from swim_b200.study import run_sweep_point
    n = 500
    base = dict(n_nodes=n, seed=404, churn_ppm=8000, rejoin_min=3, rejoin_max=11)
    nbr = generate_topology("ring", n, 32, 16, seed=2)
    from swim_b200.sim import Simulator
    sim = Simulator(default_config(suspicion_rounds=2, **base))
    sim.set_view(nbr)
    sim.save()
    for S, smax, ppm in ((2, 0, 8000), (5, 0, 8000), (3, 11, 8000), (4, 0, 30000)):
        sim.load()
        sim.set_params(suspicion_rounds=S, suspicion_max=smax, churn_ppm=ppm)
        orc = Oracle(default_config(suspicion_rounds=S, suspicion_max=smax, **{**base, "churn_ppm": ppm}))
        orc.set_view(nbr)
        res = run_sweep_point(sim, None, 40, sample_every=20)
        orc.step(40)
        assert_same_state(sim, orc, f"S {S} max {smax} ppm {ppm}")
        assert res["mismatch_series"][-1][1] == orc.mismatches()
    with pytest.raises(SwimError):
        sim.set_params(pb_cap=4)
    with pytest.raises(SwimError):
        sim.set_params(suspicion_rounds=7, suspicion_max=3)


def test_step_observe_equals_step_plus_observe():
    """swim_sim_step_observe: one call = rounds + counters + convergence count, delivered through mapped host memory."""
    rng = np.random.default_rng(12)
    n = 300
    cfg = default_config(n_nodes=n, seed=8)
    nbr = generate_topology("ring", n, 32, 16, seed=3)
    sim, orc = make_pair(cfg, nbr)
    ev = random_events(rng, n, 30, n_crash=20, n_rejoin=5, n_inject=10)
    sim.inject(ev)
    orc.inject(ev)
    for chunk in (1, 1, 1, 5, 1, 12, 1):
        c, mm = sim.step_observe(chunk)
        orc.step(chunk)
        assert c.tolist() == orc.counters().tolist() and mm == orc.mismatches(), sim.round
    assert_same_state(sim, orc, "after step_observe calls")


# ---------------------------------------------------------------- round_kernel_x: one grid barrier per round
def _xmode_case(n, topo, deg, loss, chunks, P=1, flags=0, smax=0, seed=77):
    cfg = default_config(n_nodes=n, k_indirect=3, fanout=4, pb_cap=8, suspicion_rounds=5, retransmit=8, seed=seed + n,
                         loss_ppm=loss, flags=flags)
    cfg.probes_per_round = P
    if smax:
        cfg.suspicion_max = smax
    nbr = generate_topology(topo, n, 32, deg, seed=5)
    sim, orc = make_pair(cfg, nbr)
    rng = np.random.default_rng(n)
    ev = crash_events(3, np.sort(rng.choice(n, size=max(2, n // 50), replace=False)).astype(np.uint32))
    sim.inject(ev)
    orc.inject(ev)
    for c in chunks:
        sim.step(c)
        orc.step(c)
        assert_same_state(sim, orc, f"after {c} more rounds")
    sim.close()


@pytest.mark.parametrize("xmode", ["1", "0"])
@pytest.mark.parametrize("case", [
    dict(n=1200, topo="ring", deg=24, loss=0, chunks=[2, 45, 1, 70]),           # dissemination: mail every round
    dict(n=1500, topo="random", deg=24, loss=0, chunks=[2, 150]),               # sparse knowledge, batched quiet scans behind it
    dict(n=900, topo="ring", deg=16, loss=30000, chunks=[2, 50]),               # loss: every node depends on its draws
    dict(n=900, topo="ring", deg=20, loss=0, chunks=[2, 50], P=3),
    dict(n=900, topo="ring", deg=20, loss=0, chunks=[2, 50], flags=A.F_ROUND_ROBIN | A.F_STRICT_OVERRIDE, smax=12),
])
def test_one_barrier_round_kernel(case, xmode, monkeypatch):
    """round_kernel_x (SWIM_XMODE=1: every fused launch; the default takes it for launches of >= 32 rounds on one shard)
    against the oracle on long event-free stretches — mail applied behind the barrier by the warp that owns the node,
    tentative tick decisions corrected, work lists extended while they are walked — and the same cases on the two-phase
    round_kernel (SWIM_XMODE=0)."""
    monkeypatch.setenv("SWIM_XMODE", xmode)
    _xmode_case(**case)


@pytest.mark.parametrize("world", [2, 3])
def test_one_barrier_round_kernel_sharded(world, monkeypatch):
    monkeypatch.setenv("SWIM_XMODE", "1")
    monkeypatch.setenv("SWIM_ROUND_KERNEL", "1")
    run_sharded(world, n=403, chunks=[1, 1, 3, 40], loss=0, deg=24)
    run_sharded(world, n=300, chunks=[2, 30], loss=20000, deg=20)


# ---------------------------------------------------------------- edge shapes (empty, ragged, minimal, everybody down)
def test_edge_shapes():
    """A single node with an empty view; two nodes of which one crashes; every process down; ragged rows (0..6 members) with
    the smallest parameters the config allows (k = 0, fan-out 1, one-record buffers, S = T = 1) — single-round and
    multi-round launches, every array against the oracle."""
    no = 0xFFFFFFFF

    def run(cfg, nbr, ev, chunks):
        sim, orc = make_pair(cfg, nbr)
        if ev is not None:
            sim.inject(ev)
            orc.inject(ev)
        for c in chunks:
            sim.step(c)
            orc.step(c)
            assert_same_state(sim, orc, f"after {c} more rounds")
        sim.close()

    run(default_config(n_nodes=1, seed=5), np.full((1, 32), no, dtype=np.uint32), None, [1, 40])
    nbr = np.full((2, 32), no, dtype=np.uint32)
    nbr[0, 0], nbr[1, 0] = 1, 0
    run(default_config(n_nodes=2, seed=9), nbr, crash_events(3, [1]), [1, 1, 1, 1, 40, 40])
    n = 300
    run(default_config(n_nodes=n, seed=11), generate_topology("random", n, 32, 10, seed=2), crash_events(2, list(range(n))), [1, 1, 50])
    rng = np.random.default_rng(3)
    nbr = np.full((n, 32), no, dtype=np.uint32)
    for i in range(n):
        m = np.sort(rng.choice([x for x in range(n) if x != i], size=i % 7, replace=False))
        nbr[i, :len(m)] = m
    run(default_config(n_nodes=n, seed=12, k_indirect=0, fanout=1, pb_cap=1, suspicion_rounds=1, retransmit=1), nbr,
        crash_events(2, list(range(0, n, 5))), [1, 1, 1, 60])
