"""swim_b200/daemon.py — the real-time single-node daemon (SURVEY §8(f)-3, Core.main completed) — on loopback UDP, with the
library's scalar calls running on the SIMT emulator (tests/emu; the same test on hardware is tests/test_gpu_zz_daemon.py)."""
import socket
import time

from daemon_scenarios import scenario_live_cluster_detects_a_crash, scenario_probe_escalation_and_relay  # noqa: E402
from emu_fixtures import emu_library  # noqa: F401  (autouse fixtures)


def test_probe_escalation_and_relay():
    scenario_probe_escalation_and_relay()


def test_live_cluster_detects_a_crash():
    scenario_live_cluster_detects_a_crash(period=0.25)
