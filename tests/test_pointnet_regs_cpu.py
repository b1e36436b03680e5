"""CPU: no instantiation of the TF32 PointNet kernel spills registers.

The kernel keeps its layer-2 and layer-3 A operands in registers (up to 128 per thread at C2 = 256), so its shape is
set by the register budget.  A spill would not change a result, only put local-memory traffic on the hot path, so
this compiles `pointnet_tc.cu` with the library's flags and `-Xptxas -v` and reads ptxas's report for every
`pointnet_tc_kernel` instantiation.  Skipped when no nvcc is installed.
"""
import os
import re
import subprocess

import pytest

from frustum_convnet_b200 import build


def _nvcc():
    try:
        return build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc is not installed")


def _ptxas_reports(log):
    """{mangled kernel name: ptxas report lines} from an `-Xptxas -v` log."""
    reports, name = {}, None
    for ln in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", ln)
        if m:
            name = m.group(1)
            reports[name] = []
        elif name is not None:
            reports[name].append(ln)
    return reports


def test_pointnet_tc_no_spills(tmp_path):
    nvcc = _nvcc()
    obj = str(tmp_path / "pointnet_tc.o")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "pointnet_tc.cu"),
                        "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    reports = {k: v for k, v in _ptxas_reports(r.stdout + r.stderr).items() if "pointnet_tc_kernel" in k}
    assert len(reports) == 5, sorted(reports)   # 1-CTA (64|128|256 channels) + 2-CTA clusters (128|256)
    for name, lines in reports.items():
        text = "\n".join(lines)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", text)
        assert m, name + ": no spill report\n" + text
        assert (int(m.group(1)), int(m.group(2))) == (0, 0), name + ": " + m.group(0)
