"""The NCCL stand-in on the GPU. TEST INFRASTRUCTURE ONLY. tests/emu/fake_nccl.cpp, the in-process NCCL of the emulated
tests, built against the real CUDA runtime: the ranks of a sharded run are handles of one process, one host thread each,
all on one device, and the staged exchange (K1b's buckets, the bucket counts and envelopes moved between ranks,
deliver_kernel, K2's reads of the received envelopes, and the collectives between steps) runs on the H100 without a
second GPU. A module that imports `fake_nccl_gpu` and names it (or `staged`) gets SWIM_NCCL_LIB set to the stand-in."""
import os
import shutil
import struct
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emu", "fake_nccl.cpp")
STAND_IN_TAG = 0x5157494D  # the high word of every unique id the stand-in hands out


def _nvcc():
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc")
    if not nvcc and os.path.exists("/usr/local/cuda/bin/nvcc"):
        nvcc = "/usr/local/cuda/bin/nvcc"
    return nvcc


@pytest.fixture(scope="session")
def fake_nccl_gpu_lib(tmp_path_factory):
    """Build the stand-in once per session into a temporary directory. The CUDA runtime is linked statically and its
    symbols are kept out of the library's exports, so the stand-in's runtime is its own and only the nccl* entry points
    are visible to the process."""
    nvcc = _nvcc()
    if not nvcc:
        pytest.fail("nvcc is needed to build the NCCL stand-in for the staged-exchange tests")
    so = tmp_path_factory.mktemp("fake_nccl") / "libfake_nccl.so"
    cmd = [nvcc, "-O1", "-std=c++17", "-arch=sm_90a", "-shared", "-cudart", "static", "-Xcompiler", "-fPIC,-pthread",
           "-Xlinker", "--exclude-libs,ALL", "-x", "c++", SRC, "-o", str(so)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        pytest.fail("build of the NCCL stand-in failed:\n" + r.stderr[-2000:])
    return str(so)


@pytest.fixture
def fake_nccl_gpu(fake_nccl_gpu_lib, monkeypatch):
    """SWIM_NCCL_LIB -> the stand-in, and a check that the library bound it: NCCL is bound once per process, so a test
    that ran real NCCL earlier in this process leaves it bound, and then ranks of one process on one device cannot
    form a communicator."""
    monkeypatch.setenv("SWIM_NCCL_LIB", fake_nccl_gpu_lib)
    from swim_b200.sim import nccl_unique_id
    uid = nccl_unique_id()
    if struct.unpack_from("<Q", uid)[0] >> 32 != STAND_IN_TAG:
        pytest.fail("the library bound a real NCCL before the stand-in (NCCL is bound once per process); run the "
                    "staged-exchange tests in a process that has not used NCCL")
    return fake_nccl_gpu_lib


def staged_too(argvalues, ids):
    """Parameters for "<args>,mode": each case over peer memory ("p2p") under the id it has always had, then each again
    over the staged exchange ("nccl", the id with "-nccl" appended)."""
    vals = [v if isinstance(v, tuple) else (v,) for v in argvalues]
    return [pytest.param(*v, "p2p", id=i) for v, i in zip(vals, ids)] + \
           [pytest.param(*v, "nccl", id=f"{i}-nccl") for v, i in zip(vals, ids)]
