"""The sharded code paths on ONE GPU: world 2 and 4 with every rank's handle in this process and on device 0. Ranks of one
process connect through raw device pointers (no CUDA IPC inside a process), so K1b's stores into the owner's arrays, the
cross-rank barrier (st.release.sys / ld.acquire.sys on the round words) and K2's snapshot pulls run exactly as across an
NVLink box — minus the link. Small shards: all ranks' kernels must be resident together (a rank's kernel waits for its
peers on the device). What a 1-GPU `-m gpu` run can check of SURVEY 8(e); tests/test_gpu_dist.py is the
multi-GPU form."""
import pytest

from helpers import run_sharded
from nccl_fixtures import fake_nccl_gpu, fake_nccl_gpu_lib  # noqa: F401  (fixtures)
from swim_b200 import _abi as A

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("path", ["split", "round_kernel", "nccl"])
@pytest.mark.parametrize("world", [2, 4])
def test_shards_on_one_device_equal_the_oracle(world, path, monkeypatch, request):
    """Over peer memory (split or round_kernel) and through the staged exchange ("nccl": the in-process NCCL stand-in of
    tests/nccl_fixtures.py, which needs no co-residency: the host synchronises between K1b and K2)."""
    if path == "nccl":
        request.getfixturevalue("fake_nccl_gpu")
    monkeypatch.setenv("SWIM_ROUND_KERNEL", "1" if path == "round_kernel" else "0")
    run_sharded(world, n=1201, chunks=[1] * 6 + [14, 30], loss=20000, deg=24, devices=[0] * world,
                mode="nccl" if path == "nccl" else "p2p")


def test_shards_on_one_device_variants(monkeypatch):
    monkeypatch.setenv("SWIM_ROUND_KERNEL", "1")
    run_sharded(2, n=600, chunks=[1, 1, 60], loss=0, deg=20, flags=A.F_STRICT_OVERRIDE | A.F_ROUND_ROBIN, devices=[0, 0])


def test_shards_on_one_device_sparse_knowledge():
    """Sparse views: most cross-shard envelopes are dropped at the sender by the membership filter; the few delivered ones
    go through the peer-memory path. (Shards stay small here: on ONE device every rank's pre-launched kernels hold CTA
    slots while they wait for their peers, and a rank whose next kernel finds no free slot can never publish — with
    1000 nodes per rank x 4 ranks this test dead-locked until the 60 s watchdog fired. A GPU per rank has no such limit.)"""
    run_sharded(4, n=1600, chunks=[2, 6, 12], loss=0, deg=6, devices=[0] * 4)
