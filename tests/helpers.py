"""Shared helpers for the parity tests: build the same scenario on the CUDA library (through
the C ABI) and on the CPU oracle, and compare every state array bit for bit."""
import threading

import numpy as np

from swim_b200 import _abi as A
from swim_b200.sim import concat_events, crash_events, default_config, generate_topology, make_events  # noqa: F401


def make_pair(cfg, nbr):
    from oracle.oracle import Oracle
    from swim_b200.sim import Simulator
    sim = Simulator(cfg)
    sim.set_view(nbr)
    orc = Oracle(cfg)
    orc.set_view(nbr)
    return sim, orc


def assert_same_state(sim, orc, where=""):
    for arr in range(A.ARR_COUNT):
        a, b = sim.get_array(arr), orc.get_array(arr)
        if not np.array_equal(a, b):
            idx = np.flatnonzero(a != b)[:8]
            raise AssertionError(f"{where}: array {A.ARRAY_NAMES[arr]} differs at {idx.tolist()}: "
                                 f"cuda={a[idx].tolist()} oracle={b[idx].tolist()}")
    ca, cb = sim.counters(), orc.counters()
    assert ca.tolist() == cb.tolist(), f"{where}: counters differ cuda={dict(zip(A.CTR_NAMES, ca.tolist()))} " \
                                       f"oracle={dict(zip(A.CTR_NAMES, cb.tolist()))}"
    assert sim.digest() == orc.digest(), f"{where}: digest differs"
    assert sim.mismatches() == orc.mismatches(), f"{where}: mismatch count differs"


def random_events(rng, n_nodes, rounds, n_crash, n_rejoin=0, n_inject=0):
    """A seeded event trace: crashes, later rejoins of some crashed nodes, injected messages."""
    evs = []
    crashed = rng.choice(n_nodes, size=min(n_crash, n_nodes), replace=False)
    cr = rng.integers(1, max(2, rounds // 2), size=len(crashed))
    evs.append(make_events(cr.astype(np.uint32), crashed.astype(np.uint32), np.full(len(crashed), A.EV_CRASH, np.uint8)))
    if n_rejoin:
        who = rng.choice(len(crashed), size=min(n_rejoin, len(crashed)), replace=False)
        rr = cr[who] + rng.integers(1, max(2, rounds // 2), size=len(who))
        evs.append(make_events(rr.astype(np.uint32), crashed[who].astype(np.uint32),
                               np.full(len(who), A.EV_REJOIN, np.uint8)))
    if n_inject:
        evs.append(make_events(rng.integers(1, rounds, size=n_inject).astype(np.uint32),
                               rng.integers(0, n_nodes, size=n_inject).astype(np.uint32),
                               np.full(n_inject, A.EV_INJECT, np.uint8),
                               msg_kind=rng.choice([A.MSG_SUSPECT, A.MSG_ALIVE, A.MSG_DEAD], size=n_inject).astype(np.uint8),
                               msg_node=rng.integers(0, n_nodes, size=n_inject).astype(np.uint32),
                               msg_inc=rng.integers(0, 4, size=n_inject).astype(np.int64),
                               msg_from=rng.integers(0, n_nodes, size=n_inject).astype(np.uint32)))
    return concat_events(evs)


def run_sharded(world, n, chunks, loss, deg, flags=0, mode="p2p", devices=None, churn=None, **overrides):
    """`world` handles in ONE process — on the emulator `world` emulated GPUs, on hardware all ranks on one device (or
    devices[r]): ranks of one process connect through raw device pointers (swim_sim_ipc_export / _connect), so the peers'
    arrays are addressed exactly as over NVLink. Each rank steps on its own host thread (its kernels wait for the others
    on the device); the sum of the shards must be the single-shard oracle's state. `overrides` replace config fields
    (view_cap, k_indirect, fanout, pb_cap, ...); the view is generated at that view_cap."""
    from oracle.oracle import Oracle
    from swim_b200.sim import Simulator
    rng = np.random.default_rng(world * 100 + n)
    kw = dict(n_nodes=n, k_indirect=3, fanout=4, pb_cap=6, suspicion_rounds=4, retransmit=5, loss_ppm=loss, seed=4242, flags=flags)
    if churn:
        kw.update(churn_ppm=churn[0], rejoin_min=churn[1], rejoin_max=churn[2])
    kw.update(overrides)
    nbr = generate_topology("random", n, kw.get("view_cap", 32), deg, seed=6)
    total = sum(chunks)
    events = random_events(rng, n, total, n_crash=max(2, n // 12), n_rejoin=max(1, n // 40), n_inject=n // 10)
    sims = [Simulator(default_config(rank=r, world=world, device=(devices[r] if devices else -1), **kw)) for r in range(world)]
    for s in sims:
        s.set_view(nbr)
    if mode == "p2p":
        blobs = [s.ipc_export() for s in sims]
        for s in sims:
            s.ipc_connect(blobs)
    else:  # staged exchange: NCCL replaced by tests/emu/fake_nccl.cpp (ranks = threads); the rendezvous blocks until all joined
        from swim_b200.sim import nccl_unique_id
        uid = nccl_unique_id()
        ts = [threading.Thread(target=s.connect, args=(uid,)) for s in sims]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
    for s in sims:
        s.inject(events)
    ref = Oracle(default_config(**kw))
    ref.set_view(nbr)
    ref.inject(events)
    for c in chunks:
        errs = []

        def work(s):
            try:
                s.step(c)
            except Exception as e:  # noqa: BLE001
                errs.append(e)
        ts = [threading.Thread(target=work, args=(s,)) for s in sims]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        assert not errs, errs
        ref.step(c)
        assert sum(s.digest() for s in sims) % 2 ** 64 == ref.digest(), f"digest differs at round {ref.round}"
        assert sum(s.mismatches() for s in sims) == ref.mismatches()
    assert np.sum([s.counters() for s in sims], axis=0).tolist() == ref.counters().tolist()
    for a in range(A.ARR_COUNT):
        got = sims[0].get_array(a) if a in A.REPLICATED_ARRAYS else np.concatenate([s.get_array(a) for s in sims])
        assert np.array_equal(got, ref.get_array(a)), A.ARRAY_NAMES[a]
    assert ref.counters()[A.CTR_MSGS_RECV] > 0
    for s in sims:
        s.close()
