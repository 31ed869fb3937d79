"""Sharded runs at every row width and buffer size on the SIMT emulator (tests/emu): the shapes of
sharded_shape_scenarios.py on the four sharded launch paths (round_kernel, split, round_kernel_x over peer memory, and
the staged NCCL exchange through tests/emu/fake_nccl.cpp), the calls between steps at view_cap 128 and pb_cap 32 over
both exchanges, and the staged exchange's bucket-overflow report. The H100 versions are in test_gpu_sharded_shapes.py."""
import pytest

import sharded_shape_scenarios as SS
from emu_fixtures import emu_library, fake_nccl  # noqa: F401  (autouse fixtures)

# the emulator runs the shapes at these node counts (the H100 at the shapes' own)
EMU_N = {"cap64-P2-k5f6-pb1-w3": 601, "cap128-pb32-loss-smax9-w2": 400, "cap256-P4-k7f8-churn-variants-w4": 240,
         "cap32-k0f1-pb1-w4-n13": 13}


@pytest.mark.parametrize("path", list(SS.PATHS))
@pytest.mark.parametrize("shape", list(SS.SHAPES))
def test_shape_equals_oracle(shape, path, monkeypatch):
    SS.run_shape(shape, path, monkeypatch, n=EMU_N[shape])


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
@pytest.mark.parametrize("call", SS.CALLS)
def test_between_steps_wide(call, mode):
    SS.between_steps(call, 2, 203, mode)


def test_staged_bucket_overflow_is_reported():
    SS.bucket_overflow(per=1536)
