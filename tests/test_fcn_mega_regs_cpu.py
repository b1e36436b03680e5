"""CPU: the persistent FCN kernel neither spills nor grows its stack frame.

`fcn_mega_kernel` runs 352 threads (two consumer warpgroups, the TMA, scheduler and store warps) with one CTA per
SM, which caps it at 184 registers per thread; its NT = 256 tiles keep 128 accumulator registers per thread.  A spill
or a larger stack frame would not change a result, only put local-memory traffic next to the MMAs, so this compiles
`fcn_mega.cu` with the library's flags and `-Xptxas -v` and reads ptxas's report.  The 24-byte frame is the one the
kernel had before the store warp: the six array widths the heads tile's peer replication indexes in a loop.  Skipped when no nvcc is installed.
"""
import os
import re
import subprocess

import pytest

from frustum_convnet_b200 import build

STACK_FRAME_BYTES = 24


def _nvcc():
    try:
        return build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc is not installed")


def test_fcn_mega_no_spills_no_stack_growth(tmp_path):
    nvcc = _nvcc()
    obj = str(tmp_path / "fcn_mega.o")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "fcn_mega.cu"),
                        "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    log = (r.stdout + r.stderr).splitlines()
    start = [i for i, ln in enumerate(log) if re.search(r"Compiling entry function '\S*fcn_mega_kernel\S*'", ln)]
    assert len(start) == 1, "\n".join(log)
    report = "\n".join(log[start[0] + 1: start[0] + 5])
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", report)
    assert m, "no spill report\n" + report
    frame, st, ld = (int(g) for g in m.groups())
    assert (st, ld) == (0, 0), m.group(0)
    assert frame <= STACK_FRAME_BYTES, m.group(0)
    regs = re.search(r"Used (\d+) registers", report)
    assert regs and int(regs.group(1)) <= 184, report
