"""Sharded runs at every row width and buffer size on the H100, all ranks in this process and on device 0: the shapes of
sharded_shape_scenarios.py on the four sharded launch paths, the calls between steps at view_cap 128 and pb_cap 32 over
both exchanges, and the staged exchange's bucket-overflow report. The staged exchange runs through the in-process NCCL
stand-in (tests/nccl_fixtures.py), so its device code (K1b's buckets, deliver_kernel, K2's reads of the received
envelopes) and the NCCL form of the collectives between steps run on one GPU. The emulator versions are in
test_emu_sharded_shapes.py.

Over peer memory, every rank's round kernel waits for its peers on the device, so the ranks' grids must be resident at
once (test_gpu_shards_one_device.py explains why): the shapes keep ceil(n / world) at a few hundred, and each p2p case
checks that the ranks' CTAs fit one per SM before it starts."""
import os
import re

import pytest

import sharded_shape_scenarios as SS
from nccl_fixtures import fake_nccl_gpu, fake_nccl_gpu_lib  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

DEVICE_CUH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "swim_b200", "csrc",
                          "swim_device.cuh")


def warps_per_block():
    with open(DEVICE_CUH) as f:
        return int(re.search(r"#define SWIM_WARPS_PER_BLOCK (\d+)", f.read()).group(1))


def assert_coresident(n, world):
    """One warp per node and kWarpsPerBlock warps per CTA: with at most one CTA per SM over all ranks, every rank's grid
    is resident whatever else the SM holds."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    wpb = warps_per_block()
    ctas = sum(-(-c // wpb) for c in SS.local_counts(n, world))
    assert ctas <= sms, f"{world} ranks of {n} nodes need {ctas} CTAs at once; the device has {sms} SMs"


def prepare(mode, n, world, request):
    if mode == "nccl":
        request.getfixturevalue("fake_nccl_gpu")
    else:
        assert_coresident(n, world)


@pytest.mark.parametrize("path", list(SS.PATHS))
@pytest.mark.parametrize("shape", list(SS.SHAPES))
def test_shape_equals_oracle(shape, path, monkeypatch, request):
    s = SS.SHAPES[shape]
    prepare(SS.PATHS[path][0], s["n"], s["world"], request)
    SS.run_shape(shape, path, monkeypatch, devices=[0] * s["world"])


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
@pytest.mark.parametrize("call", SS.CALLS)
def test_between_steps_wide(call, mode, monkeypatch, request):
    monkeypatch.setenv("SWIM_ROUND_KERNEL", "1")
    prepare(mode, 800, 2, request)
    SS.between_steps(call, 2, 800, mode, devices=[0, 0])


def test_staged_bucket_overflow_is_reported(fake_nccl_gpu):  # noqa: F811
    SS.bucket_overflow(per=1536, devices=[0] * 4)
