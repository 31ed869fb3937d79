"""Sharded runs away from the default configuration shape, shared by the emulator tests (test_emu_sharded_shapes.py) and
the H100 tests (test_gpu_sharded_shapes.py).

Every sharded kernel has an instance per row width W (view_cap / 32), the staged envelope is 1 + pb_cap uint4 wide, the
peer snapshot pull is strided by pb_cap, and the receiver lists and exchange buckets are sized from fanout. The default
shape (view_cap 32, k 3, fanout 4, pb_cap 6, one probe per round) hides a stride or width bug that is only right there. The
shapes below put every one of these values at an edge at least once; each runs on the four sharded launch paths and is
held to the single-shard oracle after every chunk of rounds (sharded_edit_scenarios.Shards.check: every array, the
digest, the counter sums and the mismatch sums)."""
import numpy as np

import sharded_edit_scenarios as SE
from helpers import make_events
from swim_b200 import _abi as A

# id -> world, n, view degree, chunks, config overrides
SHAPES = {
    # n not a multiple of world (shards of 201, 201, 199 rows: the second and third start off a multiple of 4), two probes
    # per round, one-record buffers
    "cap64-P2-k5f6-pb1-w3": dict(world=3, n=601, deg=48, chunks=(1, 1, 1, 4, 13),
                                 kw=dict(view_cap=64, probes_per_round=2, k_indirect=5, fanout=6, pb_cap=1,
                                         loss_ppm=20000)),
    # the widest buffer: a staged envelope of 33 uint4, snapshots strided by 32
    "cap128-pb32-loss-smax9-w2": dict(world=2, n=800, deg=100, chunks=(1, 1, 1, 5, 12),
                                      kw=dict(view_cap=128, pb_cap=32, loss_ppm=30000, suspicion_max=9)),
    # the widest row, the largest fan-out and probe count, device churn and both protocol variants
    "cap256-P4-k7f8-churn-variants-w4": dict(world=4, n=800, deg=200, chunks=(1, 1, 1, 3, 10),
                                             kw=dict(view_cap=256, probes_per_round=4, k_indirect=7, fanout=8,
                                                     churn_ppm=30000, rejoin_min=2, rejoin_max=6, loss_ppm=10000,
                                                     flags=A.F_STRICT_OVERRIDE | A.F_ROUND_ROBIN)),
    # no proxies, one recipient, one-record buffers; shards of 4, 4, 4 and 1 rows
    "cap32-k0f1-pb1-w4-n13": dict(world=4, n=13, deg=6, chunks=(1, 1, 2, 4, 12),
                                  kw=dict(view_cap=32, k_indirect=0, fanout=1, pb_cap=1, loss_ppm=20000)),
}

# launch path -> (exchange, environment). p2p: ranks connected over peer memory (raw device pointers within a process);
# staged: NCCL (the in-process stand-in), split launches with deliver_kernel between K1b and K2.
PATHS = {
    "round_kernel": ("p2p", {"SWIM_ROUND_KERNEL": "1", "SWIM_XMODE": "0"}),
    "split": ("p2p", {"SWIM_ROUND_KERNEL": "0"}),
    "round_kernel_x": ("p2p", {"SWIM_ROUND_KERNEL": "1", "SWIM_XMODE": "1"}),
    "staged": ("nccl", {}),
}


def local_counts(n, world):
    """Rows per rank: rank r holds [r * per, min(n, (r + 1) * per)), per = ceil(n / world)."""
    per = -(-n // world)
    return [max(0, min(n, (r + 1) * per) - r * per) for r in range(world)]


def use_path(path, monkeypatch):
    mode, env = PATHS[path]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    return mode


def run_shape(shape, path, monkeypatch, devices=None, n=None):
    """One shape on one launch path against the oracle after every chunk; `n` replaces the shape's node count."""
    s = SHAPES[shape]
    mode = use_path(path, monkeypatch)
    n = n or s["n"]
    sh, orc = SE.setup(s["world"], n, s["deg"], mode, seed=21, devices=devices, rounds=sum(s["chunks"]), **s["kw"])
    SE.step(sh, orc, s["chunks"])
    assert orc.counters()[A.CTR_MSGS_RECV] > 0
    sh.close()


# ------------------------------------------------------------------ the calls between steps at cap 128, pb_cap 32
WIDE = dict(view_cap=128, pb_cap=32)


def between_steps(call, world, n, mode, devices=None):
    import join_scenarios as JS
    import leave_scenarios as LS
    if call == "push_pull":
        SE.push_pull_every(world, n, mode, rounds=24, every=6, devices=devices, **WIDE)
    elif call == "join":
        JS.sharded_joins(world, n, mode, devices=devices, **WIDE)
    elif call == "leave":
        LS.sharded_leaves(world, n, mode, devices=devices, **WIDE)
    else:  # remove / add
        SE.remove_dead_then_rounds(world, n, mode, devices=devices, **WIDE)
        SE.add_members_then_rounds(world, n, mode, devices=devices, deg=120, **WIDE)


CALLS = ["push_pull", "join", "leave", "remove_add"]


# ------------------------------------------------------------------ staged bucket overflow
def bipartite_view(n, world, cap, deg):
    """Ranks paired (0, 1), (2, 3), ...: local node i of one rank of a pair lists local nodes i .. i + deg - 1 (mod the
    shard size) of the other, and is listed by exactly those: the view is symmetric, and every envelope a node sends goes
    to the other rank of its pair."""
    per = n // world
    nbr = np.full((n, cap), A.NO_MEMBER, dtype=np.uint32)
    i = np.arange(per)
    for a in range(0, world, 2):
        b = a + 1
        for j in range(deg):
            nbr[a * per + i, j] = b * per + (i + j) % per
            nbr[b * per + i, j] = a * per + (i - j) % per
    nbr[:, :deg].sort(axis=1)
    return nbr


def bucket_overflow(per, devices=None):
    """World 4, fan-out 8, staged exchange. Every node of rank 0 hears a Suspect about itself in round 1 and refutes it,
    so in that round it sends an Alive about itself to 8 members of its view, all of them on rank 1, all of which list
    it: 8 * per envelopes for the rank-1 bucket, whose capacity is 2 * (per * 8 / 4) + 4096. The overflow is reported as
    SWIM_ECAP by every rank in the same call (the counts are all-gathered before anything moves); the next step on each
    handle is refused with SWIM_ESTATE, and the handles close."""
    from swim_b200._lib import SwimError
    world, fanout = 4, 8
    n = world * per
    assert fanout * per > 2 * (per * fanout // world) + 4096, "the rank-1 bucket must be too small"
    kw = SE.config(n, 31, view_cap=32, k_indirect=7, fanout=fanout, probes_per_round=1, loss_ppm=0)
    sh = SE.Shards(world, kw, bipartite_view(n, world, 32, 16), "nccl", devices)
    nodes = np.arange(per, dtype=np.uint32)
    sh.inject(make_events(np.ones(per, np.uint32), nodes, np.full(per, A.EV_INJECT, np.uint8),
                          msg_kind=np.full(per, A.MSG_SUSPECT, np.uint8), msg_node=nodes,
                          msg_inc=np.zeros(per, np.int64), msg_from=nodes + per))

    def step(s):
        try:
            s.step(1)
            return A.OK, ""
        except SwimError as e:
            return e.code, str(e)
    got = sh.all(step)  # round 1
    assert [c for c, _ in got] == [A.ECAP] * world, got
    assert all("rank 0 overflowed an exchange bucket" in m for _, m in got), got
    assert [c for c, _ in sh.all(step)] == [A.ESTATE] * world
    sh.close()
