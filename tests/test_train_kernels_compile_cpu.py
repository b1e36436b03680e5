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
    "train_fwd_kernel<false>", "train_fwd_finish_kernel<false>", "train_reduce_kernel<false>", "train_dw_kernel<false>",
    "train_dx_kernel<false>", "train_pool_fwd_kernel", "train_pool_bwd_kernel", "train_finalize_kernel",
    "train_adam_kernel", "train_fwd_plain_kernel<false>", "train_dx_plain_kernel", "train_dw_plain_kernel<false>",
]


def _nvcc():
    try:
        return build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc is not installed")


def kernel_key(mangled):
    """_ZN3fcn<length><name>E... -> name, and _ZN3fcn<length><name>ILb0EE... -> name<false> (ILb1E: name<true>):
    the two instantiations of a `template <bool>` kernel are told apart."""
    m = re.match(r"_ZN3fcn(\d+)", mangled)
    if not m:
        return None
    end = m.end() + int(m.group(1))
    t = re.match(r"ILb([01])E", mangled[end:])
    return mangled[m.end():end] + ("<%s>" % ("true" if t.group(1) == "1" else "false") if t else "")


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
    for mangled, usage in res.items():
        k = kernel_key(mangled)
        if k:
            by_name[k] = usage
    missing = [k for k in KERNELS if k not in by_name]
    assert not missing, "kernels not compiled: %s (found %s)" % (missing, sorted(by_name))
    for k in KERNELS:
        assert by_name[k] == (0, 0, 0), "%s: %d-byte stack frame, %d / %d bytes of spill stores / loads" % (
            (k,) + by_name[k])
