"""Register budget of the per-round kernels (CPU only: ptxas runs without a GPU).

The round kernels are launched at __launch_bounds__(kThreads, kMinBlocks): 64 registers per thread, so that 32 warps per SM
are resident and the grid barrier's one-wave grid holds. What does not fit goes to local memory, and every spill load
sits on a warp's serial chain through a round. This test compiles swim_sim.cu for sm_90a with `-Xptxas -v` and holds
each instantiation to the spill figures recorded below: the timed single-shard kernels of the 1 GPU benchmark at their
figures of the commit that moved the counters to shared memory and split off the single-shard instances, every other
instantiation at its figures from before that commit.
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (spill store bytes, spill load bytes) ptxas may not exceed, per kernel instantiation.
TIMED = {
    "round_kernel_x<1, false>": (1318, 2000),  # rounds 10.. of bench.py's 448-round window (was 3042 / 4516)
    "round_kernel<1, false>": (566, 728),      # rounds 6..9, and the 20-round window (was 1054 / 1292)
}
# before: round_kernel / round_kernel_x had one instance per W, for single-shard and sharded launches alike
OLD_ROUND = {"round_kernel": {1: (1054, 1292), 2: (1296, 1528), 4: (1864, 2268), 8: (2900, 4216)},
             "round_kernel_x": {1: (3042, 4516), 2: (2634, 3476), 4: (3710, 4960), 8: (5444, 8352)}}
OTHERS = {
    "tick_scan_kernel": {1: (0, 0), 2: (104, 112), 4: (168, 144), 8: (232, 160)},
    "tick_work_kernel": {1: (104, 72), 2: (226, 216), 4: (358, 336), 8: (582, 1248)},
    "recv_kernel": {1: (0, 0), 2: (28, 36), 4: (92, 88), 8: (264, 288)},
}
REG_CAP = 64


def budget():
    out = dict(TIMED)
    for name, per_w in OLD_ROUND.items():
        for w, lim in per_w.items():
            for sharded in ("false", "true"):
                out.setdefault(f"{name}<{w}, {sharded}>", lim)
    for name, per_w in OTHERS.items():
        for w, lim in per_w.items():
            out[f"{name}<{w}>"] = lim
    return out


_MANGLED = re.compile(r"_ZN4swim(\d+)(\w+?)ILi(\d+)E(?:Lb([01])E)?EEvNS_6SimDevE$")


def readable(mangled):
    m = _MANGLED.match(mangled)
    if not m or int(m.group(1)) != len(m.group(2)):
        return None
    name, w, b = m.group(2), m.group(3), m.group(4)
    return f"{name}<{w}>" if b is None else f"{name}<{w}, {'true' if b == '1' else 'false'}>"


def parse_ptxas(text):
    """{kernel: (registers, stack bytes, spill store bytes, spill load bytes)} of the swim:: round kernels in -Xptxas -v output."""
    res, cur, props = {}, None, {}
    for line in text.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            props[cur] = tuple(int(x) for x in m.groups())
            continue
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and cur in props:
            name = readable(cur)
            if name:
                res[name] = (int(m.group(1)),) + props[cur]
    return res


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if not nvcc:
        pytest.skip("nvcc not found")
    from swim_b200 import build as b
    out = tmp_path_factory.mktemp("ptxas") / "swim_sim.o"
    cmd = [nvcc, "-Xptxas", "-v"] + b.NVCC_FLAGS + ["-x", "cu", "-c", os.path.join(b.CSRC, "swim_sim.cu"), "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return parse_ptxas(r.stdout + r.stderr)


def test_every_round_kernel_is_reported(ptxas_report):
    assert set(budget()) <= set(ptxas_report), sorted(set(budget()) - set(ptxas_report))


@pytest.mark.parametrize("kernel", sorted(budget()))
def test_spills_within_budget(ptxas_report, kernel):
    regs, stack, st, ld = ptxas_report[kernel]
    lim_st, lim_ld = budget()[kernel]
    assert regs <= REG_CAP, (kernel, regs)
    assert st <= lim_st and ld <= lim_ld, f"{kernel}: {st} / {ld} bytes spill stores / loads, budget {lim_st} / {lim_ld}"


def test_parse_ptxas_names():
    assert readable("_ZN4swim14round_kernel_xILi1ELb0EEEvNS_6SimDevE") == "round_kernel_x<1, false>"
    assert readable("_ZN4swim11recv_kernelILi8EEEvNS_6SimDevE") == "recv_kernel<8>"
    assert readable("_ZN4swim12event_kernelILi1EEEvNS_6SimDevEPKNS_8DevEventEjPKj") is None
