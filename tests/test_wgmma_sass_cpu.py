"""CPU: the wgmma kernels keep their MMAs asynchronous.

ptxas serializes every wgmma.mma_async of a kernel (one WARPGROUP.DEPBAR after each HGMMA, performance
advisory C7520) when an accumulator register is touched between wgmma.fence and the MMA without a fence of its
own, e.g. when the per-stage fence is missing.  Nothing fails then: results stay bit-exact and only the tensor
pipe sits idle, so this compiles the hot-path sources with the library's flags and checks the compiler's
advisories and the SASS.  Skipped when no nvcc is installed.
"""
import os
import re
import subprocess

import pytest

from frustum_convnet_b200 import build

SOURCES = ["pointnet_tc.cu", "fcn_mega.cu", "conv_gemm_tma.cu"]


def _nvcc():
    try:
        return build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc is not installed")


def _sass_functions(sass):
    """{mangled kernel name: SASS text} from `cuobjdump -sass` output."""
    parts = re.split(r"^\s*Function : (\S+)\s*$", sass, flags=re.M)
    return dict(zip(parts[1::2], parts[2::2]))


@pytest.mark.parametrize("src", SOURCES)
def test_wgmma_not_serialized(src, tmp_path):
    nvcc = _nvcc()
    obj = str(tmp_path / (src[:-3] + ".o"))
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, src), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    advisories = [ln for ln in log.splitlines() if "C7520" in ln or "C7519" in ln]
    assert not advisories, "\n".join(advisories)

    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    kernels = {name: body for name, body in _sass_functions(sass).items() if "HGMMA" in body}
    assert kernels, "no wgmma kernel found in " + src
    for name, body in kernels.items():
        n_mma = len(re.findall(r"\bHGMMA\.", body))
        n_depbar = len(re.findall(r"\bWARPGROUP\.DEPBAR\b", body))
        assert n_depbar < n_mma, "%s: %d WARPGROUP.DEPBAR for %d HGMMA (serialized)" % (name, n_depbar, n_mma)
