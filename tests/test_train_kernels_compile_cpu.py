"""CPU: the training kernels compile without a stack frame or spills.

The GEMM kernels of csrc/train.cu share force-inlined helpers that take the shared tiles and the accumulator
by reference.  Once inlined they cost nothing; a helper that ptxas cannot keep in registers puts the
accumulator on the stack instead, and nothing fails then: results stay the same and only the kernel slows
down.  So this compiles train.cu with the library's flags and reads ptxas's resource report for every
training kernel.  Skipped when no nvcc is installed.
"""
import os
import re
import subprocess

import pytest

from frustum_convnet_b200 import build

KERNELS = [
    "train_fwd_kernel", "train_fwd_finish_kernel", "train_reduce_kernel", "train_dw_kernel", "train_dx_kernel",
    "train_pool_fwd_kernel", "train_pool_bwd_kernel", "train_finalize_kernel", "train_adam_kernel",
    "train_fwd_plain_kernel", "train_dx_plain_kernel", "train_dw_plain_kernel",
]


def _nvcc():
    try:
        return build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc is not installed")


def _resources(log):
    """{mangled kernel name: (stack frame, spill stores, spill loads)} from `-Xptxas -v` output."""
    res, cur = {}, None
    for ln in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", ln)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m and cur is not None:
            res[cur] = tuple(int(v) for v in m.groups())
    return res


def test_train_kernels_no_stack_no_spills(tmp_path):
    nvcc = _nvcc()
    obj = str(tmp_path / "train.o")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "train.cu"),
                        "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    res = _resources(r.stdout + r.stderr)
    by_name = {}
    for mangled, usage in res.items():                    # _ZN3fcn<length><name>E...
        m = re.match(r"_ZN3fcn(\d+)", mangled)
        if m:
            by_name[mangled[m.end():m.end() + int(m.group(1))]] = usage
    missing = [k for k in KERNELS if k not in by_name]
    assert not missing, "kernels not compiled: %s (found %s)" % (missing, sorted(by_name))
    for k in KERNELS:
        assert by_name[k] == (0, 0, 0), "%s: %d-byte stack frame, %d / %d bytes of spill stores / loads" % (
            (k,) + by_name[k])
