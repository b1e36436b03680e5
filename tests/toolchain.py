"""The CPU tests' compilers: each CUDA source of the library compiled once per process with the library's flags and
ptxas's resource report, its SASS, and g++ builds of the host-compilable device headers.

Every check on ptxas's report or on the SASS reads it through `compile_cuda`, so the report is parsed in one place,
and a report that stops parsing (ptxas rewords a line) fails every check instead of leaving one with nothing to
compare."""
import atexit
import ctypes
import functools
import os
import re
import shutil
import subprocess
import tempfile
from typing import NamedTuple

import pytest

from frustum_convnet_b200 import build

_TMP = tempfile.mkdtemp(prefix="fcn_toolchain_")
atexit.register(shutil.rmtree, _TMP, ignore_errors=True)


def nvcc():
    try:
        return build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc is not installed")


@functools.lru_cache(maxsize=None)
def nvcc_release():
    """'12.9' for CUDA 12.9."""
    out = subprocess.run([nvcc(), "--version"], capture_output=True, text=True, check=True).stdout
    return re.search(r"release (\d+\.\d+)", out).group(1)


class Kernel(NamedTuple):
    """ptxas's resource report of one entry function; sizes in bytes."""
    registers: int
    stack: int
    spill_stores: int
    spill_loads: int
    report: str

    @property
    def local_memory(self):
        """(stack frame, spill stores, spill loads)."""
        return self.stack, self.spill_stores, self.spill_loads


_ENTRY = re.compile(r"Compiling entry function '(\S+)' for 'sm_90a'")


def _kernels(log):
    parts = _ENTRY.split(log)
    kernels = {}
    for name, report in zip(parts[1::2], parts[2::2]):
        frame = re.search(r"Function properties for %s\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                          r"(\d+) bytes spill loads" % re.escape(name), report)
        regs = re.search(r"Used (\d+) registers", report)
        assert frame and regs, "no resource report for %s in ptxas's output:\n%s" % (name, report)
        kernels[name] = Kernel(int(regs.group(1)), *(int(v) for v in frame.groups()), report)
    return kernels


class Compiled:
    """One source compiled with `-Xptxas -v`: the compiler's log, the object, and {mangled entry name: Kernel}."""

    def __init__(self, log, obj):
        self.log, self.obj = log, obj
        self.kernels = _kernels(log)

    @functools.cache
    def sass(self):
        """{mangled function name: SASS text} from `cuobjdump -sass` of the object."""
        cuobjdump = os.path.join(os.path.dirname(nvcc()), "cuobjdump")
        out = subprocess.run([cuobjdump, "-sass", self.obj], capture_output=True, text=True, check=True).stdout
        parts = re.split(r"^\s*Function : (\S+)\s*$", out, flags=re.M)
        return dict(zip(parts[1::2], parts[2::2]))


@functools.lru_cache(maxsize=None)
def compile_cuda(src):
    """csrc/<src> compiled with the library's flags and `-Xptxas -v`, once per process."""
    obj = os.path.join(_TMP, src[:-3] + ".o")
    r = subprocess.run([nvcc()] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, src),
                                                      "-o", obj], capture_output=True, text=True)
    log = r.stdout + r.stderr
    if r.returncode != 0:
        pytest.fail("nvcc failed on %s:\n%s" % (src, log))
    return Compiled(log, obj)


def kernel_key(mangled):
    """_ZN3fcn<length><name>E... -> name, and _ZN3fcn<length><name>ILb0EE... -> name<false> (ILb1E: name<true>):
    the two instantiations of a `template <bool>` kernel are told apart."""
    m = re.match(r"_ZN3fcn(\d+)", mangled)
    if not m:
        return None
    end = m.end() + int(m.group(1))
    t = re.match(r"ILb([01])E", mangled[end:])
    return mangled[m.end():end] + ("<%s>" % ("true" if t.group(1) == "1" else "false") if t else "")


def fma_cpu():
    try:
        with open("/proc/cpuinfo") as f:
            return " fma " in f.read().replace("\n", " ")
    except OSError:
        return False


@functools.lru_cache(maxsize=None)
def host_library(harness_text, flags, include_dirs=()):
    """`g++ -O2 -shared -fPIC` build of a C++ harness around a host-compilable header, loaded with ctypes; once per
    (harness, flags, include directories)."""
    d = tempfile.mkdtemp(dir=_TMP)
    src, so = os.path.join(d, "harness.cpp"), os.path.join(d, "harness.so")
    with open(src, "w") as f:
        f.write(harness_text)
    inc = [a for i in include_dirs for a in ("-I", i)]
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC"] + inc + list(flags) + ["-o", so, src])
    return ctypes.CDLL(so)
