"""CPU: the persistent FCN kernel neither spills nor grows its stack frame.

`fcn_mega_kernel` runs 352 threads (two consumer warpgroups, the TMA, scheduler and store warps) with one CTA per
SM, which caps it at 184 registers per thread; its NT = 256 tiles keep 128 accumulator registers per thread.  A spill
or a larger stack frame would not change a result, only put local-memory traffic next to the MMAs, so this compiles
`fcn_mega.cu` with the library's flags and `-Xptxas -v` and reads ptxas's report.  The 24-byte frame is the one the
kernel had before the store warp: the six array widths the heads tile's peer replication indexes in a loop.  Skipped when no nvcc is installed.
"""
from toolchain import compile_cuda

STACK_FRAME_BYTES = 24


def test_fcn_mega_no_spills_no_stack_growth():
    c = compile_cuda("fcn_mega.cu")
    found = [k for m, k in c.kernels.items() if "fcn_mega_kernel" in m]
    assert len(found) == 1, c.log
    k = found[0]
    assert (k.spill_stores, k.spill_loads) == (0, 0), k.report
    assert k.stack <= STACK_FRAME_BYTES, k.report
    assert k.registers <= 184, k.report
