"""CPU: no instantiation of the TF32 PointNet kernel spills registers.

The kernel keeps its layer-2 and layer-3 A operands in registers (up to 128 per thread at C2 = 256), so its shape is
set by the register budget.  A spill would not change a result, only put local-memory traffic on the hot path, so
this compiles `pointnet_tc.cu` with the library's flags and `-Xptxas -v` and reads ptxas's report for every
`pointnet_tc_kernel` instantiation.  Skipped when no nvcc is installed.
"""
from toolchain import compile_cuda


def test_pointnet_tc_no_spills():
    reports = {m: k for m, k in compile_cuda("pointnet_tc.cu").kernels.items() if "pointnet_tc_kernel" in m}
    assert len(reports) == 5, sorted(reports)   # 1-CTA (64|128|256 channels) + 2-CTA clusters (128|256)
    for name, k in reports.items():
        assert (k.spill_stores, k.spill_loads) == (0, 0), name + ":\n" + k.report
