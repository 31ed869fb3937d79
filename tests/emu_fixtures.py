"""The emulator fixtures of the test_emu_* modules. TEST INFRASTRUCTURE ONLY. A module that imports them has pytest
register them there, autouse included: its tests run on the library built for tests/emu's SIMT emulator, and with
fake_nccl the staged exchange binds the in-process NCCL stand-in."""
import os
import sys

import pytest

from swim_b200 import _abi as A

EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")


@pytest.fixture(scope="module", autouse=True)
def emu_library():
    import swim_b200._lib as L
    sys.path.insert(0, EMU)
    import build_emu
    so = build_emu.build()
    saved = (L.SO_PATH, L._lib)
    L.SO_PATH, L._lib = so, None
    assert L.lib().swim_abi_version() == A.ABI_VERSION
    yield
    L.SO_PATH, L._lib = saved


@pytest.fixture(autouse=True)
def fake_nccl(monkeypatch):
    monkeypatch.setenv("SWIM_NCCL_LIB", os.path.join(EMU, "libfake_nccl.so"))
