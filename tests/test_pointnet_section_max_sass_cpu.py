"""CPU: every warp of the TF32 PointNet kernel takes its section max by reduce-scatter passes over its lanes.

The passes are xor butterflies (SHFL.BFLY) and one index shuffle per section; a segmented suffix max would shift
values down the lanes (SHFL.DOWN), which no instantiation may contain.  Skipped when no nvcc is installed.
"""
import re

from toolchain import compile_cuda


def test_pointnet_tc_has_no_suffix_max():
    sass = {m: body for m, body in compile_cuda("pointnet_tc.cu").sass().items() if "pointnet_tc_kernel" in m}
    assert len(sass) == 5, sorted(sass)
    for name, body in sass.items():
        assert re.search(r"\bSHFL\.BFLY\b", body), name + ": no butterfly section max"
        assert not re.search(r"\bSHFL\.DOWN\b", body), name + ": SHFL.DOWN (segmented suffix max)"
