"""Spills of the kernels that run the per-round scan, after the scan moved from the 16-byte meta records to the 4-byte
summary word per node (CPU only: ptxas runs without a GPU). tests/test_register_budget.py holds every instantiation to
its older figures; this file holds the scanning kernels of the 1-GPU benchmark to the figures of the summary-word scan,
each strictly below the figures of the meta-record scan."""
import pytest

from test_register_budget import REG_CAP, ptxas_report  # noqa: F401  (the fixture compiles swim_sim.cu once per module)

# (spill store bytes, spill load bytes): the summary-word scan's figures, and the meta-record scan's before it
BUDGET = {
    "round_kernel_x<1, false>": ((1210, 1984), (1318, 2000)),
    "round_kernel<1, false>": ((272, 308), (566, 728)),
    "tick_scan_kernel<1>": ((0, 0), (0, 0)),
}


@pytest.mark.parametrize("kernel", sorted(BUDGET))
def test_scan_kernel_spills(ptxas_report, kernel):  # noqa: F811
    regs, _stack, st, ld = ptxas_report[kernel]
    (lim_st, lim_ld), (old_st, old_ld) = BUDGET[kernel]
    assert regs <= REG_CAP, (kernel, regs)
    assert st <= lim_st and ld <= lim_ld, f"{kernel}: {st} / {ld} bytes spill stores / loads, budget {lim_st} / {lim_ld}"
    assert (lim_st, lim_ld) == (0, 0) or (lim_st < old_st and lim_ld < old_ld)
