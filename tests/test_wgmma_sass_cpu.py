"""CPU: the wgmma kernels keep their MMAs asynchronous.

ptxas serializes every wgmma.mma_async of a kernel (one WARPGROUP.DEPBAR after each HGMMA, performance
advisory C7520) when an accumulator register is touched between wgmma.fence and the MMA without a fence of its
own, e.g. when the per-stage fence is missing.  Nothing fails then: results stay bit-exact and only the tensor
pipe sits idle, so this compiles the hot-path sources with the library's flags and checks the compiler's
advisories and the SASS.  Skipped when no nvcc is installed.
"""
import re

import pytest

from toolchain import compile_cuda

SOURCES = ["pointnet_tc.cu", "fcn_mega.cu", "conv_gemm_tma.cu"]


@pytest.mark.parametrize("src", SOURCES)
def test_wgmma_not_serialized(src):
    c = compile_cuda(src)
    advisories = [ln for ln in c.log.splitlines() if "C7520" in ln or "C7519" in ln]
    assert not advisories, "\n".join(advisories)

    kernels = {name: body for name, body in c.sass().items() if "HGMMA" in body}
    assert kernels, "no wgmma kernel found in " + src
    for name, body in kernels.items():
        n_mma = len(re.findall(r"\bHGMMA\.", body))
        n_depbar = len(re.findall(r"\bWARPGROUP\.DEPBAR\b", body))
        assert n_depbar < n_mma, "%s: %d WARPGROUP.DEPBAR for %d HGMMA (serialized)" % (name, n_depbar, n_mma)
