"""Seed joins (swim_sim_join) on the SIMT emulator (tests/emu), against the oracle after every call: single-shard
scenarios at every row width, and sharded handles of world 2 and 3 over peer memory and through the staged NCCL exchange
(tests/emu/fake_nccl.cpp). The H100 versions are in test_gpu_join.py."""
import ctypes as C
import os
import subprocess
import tempfile

import pytest

import join_scenarios as S
from swim_b200 import _abi as A
from emu_fixtures import emu_library, fake_nccl  # noqa: F401  (autouse fixtures)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_join_layout_matches_header():
    probe = r'''
#include <stdio.h>
#include <stddef.h>
#include "swim.h"
int main(void) { printf("%zu %zu %zu %d\n", sizeof(swim_join_t), offsetof(swim_join_t, node), offsetof(swim_join_t, seed),
                        SWIM_JOIN_FRESH); return 0; }'''
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "p.c"), os.path.join(d, "p")
        open(src, "w").write(probe)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
        size, node, seed, fresh = map(int, subprocess.check_output([exe], text=True).split())
    assert (size, node, seed) == (C.sizeof(A.Join), A.Join.node.offset, A.Join.seed.offset)
    assert A.JOIN_DTYPE.itemsize == size and A.JOIN_DTYPE.fields["seed"][1] == seed and fresh == A.JOIN_FRESH


@pytest.mark.parametrize("cap", [32, 64, 128, 256])
def test_every_row_width(cap):
    _, _, tot = S.join_every(160, cap, min(cap // 2 + 3, 100), rounds=18, every=6, seed=cap, loss_ppm=20000,
                             churn_ppm=5000, rejoin_min=2, rejoin_max=6)
    assert tot[0] > 0 and tot[1] > 0


@pytest.mark.parametrize("flags,suspicion_max", [(A.F_STRICT_OVERRIDE, 0), (0, 9), (A.F_ROUND_ROBIN, 0)])
def test_protocol_variants(flags, suspicion_max):
    S.join_every(140, 32, 14, rounds=24, every=4, flags=flags, suspicion_max=suspicion_max, loss_ppm=30000)


def test_edge_cases():
    S.edge_cases()


def test_hub():
    S.hub(600, 500)


def test_full_rows():
    S.full_rows()


@pytest.mark.parametrize("flags,suspicion_max", [(0, 0), (A.F_STRICT_OVERRIDE, 0), (0, 9)])
def test_refutations(flags, suspicion_max):
    S.refutations(flags=flags, suspicion_max=suspicion_max)


def test_save_join_load():
    S.save_join_load(160)


def test_export_after_join():
    S.export_after_join(80)


def test_fresh_rebuild():
    S.fresh_rebuild(400, frac=0.05)


def test_with_push_pull():
    S.with_push_pull(200)


def test_error_paths():
    S.error_paths()
    S.sharded_not_connected()


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
@pytest.mark.parametrize("world", [2, 3])
def test_sharded(world, mode):
    S.sharded_joins(world, 211, mode)


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
def test_sharded_equals_single_shard(mode):
    S.sharded_equals_single_shard(700, 3, None, mode)


def test_study_join_hosts():
    """run_sweep_point with join hosts under seeded churn: the processes that restarted in a chunk join through the hosts
    after it, on the device code and on the oracle alike (same series, counters, report and join totals)."""
    import numpy as np
    from oracle.oracle import Oracle
    from between_steps_oracle import join as oracle_join
    from swim_b200.sim import Simulator, default_config, generate_topology
    from swim_b200.study import run_sweep_point

    class JoiningOracle(Oracle):
        def join(self, nodes, seeds, fresh=False):
            return oracle_join(self, nodes, seeds, fresh)

    n = 300
    cfg = default_config(n_nodes=n, seed=21, suspicion_rounds=3, churn_ppm=20000, rejoin_min=3, rejoin_max=8)
    nbr = generate_topology("random", n, 32, 12, seed=21)
    hosts = np.array([5, 77, 200], np.uint32)
    out = []
    for h in (Simulator(cfg), JoiningOracle(cfg)):
        h.set_view(nbr)
        res = run_sweep_point(h, None, 40, 10, join_hosts=hosts, join_fresh=True)
        res["join"].pop("host_s_rank0")
        out.append({k: res[k] for k in ("mismatch_series", "counters", "report", "join")})
    assert out[0] == out[1]
    assert out[0]["join"]["pairs"] > 0 and out[0]["join"]["exchanges"] > 0 and out[0]["join"]["inserted"] > 0
