"""CPU: the deterministic training entries - compiled without a stack frame or spills, declared in _lib.py, and
sized from the layer's shape only."""
import ctypes as C
import os
import re

import pytest

from frustum_convnet_b200 import _lib, build
from toolchain import compile_cuda, kernel_key

TRAIN_KERNELS = [
    "train_fwd_kernel<true>", "train_fwd_finish_kernel<true>", "train_slots_sum_kernel", "train_reduce_kernel<true>",
    "train_dw_kernel<true>", "train_dw_sum_kernel", "train_dx_kernel<true>", "train_dx_sum_kernel",
    "train_fwd_plain_kernel<true>", "train_dw_plain_kernel<true>",
]
ENTRIES = ["fcn_train_deterministic_workspace_floats", "fcn_train_forward_deterministic",
           "fcn_train_backward_deterministic", "fcn_det_loss_deterministic_scratch_floats", "fcn_det_loss_deterministic"]


def _usage(src):
    """{kernel_key: Kernel.local_memory} of csrc/<src>."""
    return {kernel_key(m): k.local_memory for m, k in compile_cuda(src).kernels.items()}


def test_deterministic_train_kernels_no_stack_no_spills():
    res = _usage("train.cu")
    for k in TRAIN_KERNELS:
        assert res.get(k) == (0, 0, 0), "%s: %r (stack frame, bytes spilled: stores, loads)" % (k, res.get(k))


def test_deterministic_loss_kernels_compile_like_the_default():
    """The ordered row kernel is the default one's template instantiation, whose corner arrays live in a local frame:
    the same frame, and no spills."""
    res = _usage("loss.cu")
    assert res["det_loss_rows_kernel<true>"] == res["det_loss_rows_kernel<false>"]
    assert res["det_loss_rows_kernel<true>"][1:] == (0, 0)
    assert res["det_loss_slots_kernel"] == (0, 0, 0)


def test_new_entries_are_declared():
    header = open(os.path.join(build.HERE, "..", "include", "frustum_b200.h")).read()
    for name in ENTRIES:
        assert name in _lib.SIGNATURES, name
        assert re.search(r"FCN_API [^;]*\b%s\(" % name, header), name


def _layer(B, T, C_in, N, n_seg=1, has_bn=1, up=1, tap=0, stride=1):
    L = _lib.TrainLayer()
    L.B, L.T_out, L.n_seg, L.N, L.Cout, L.up, L.has_bn, L.relu = B, T, n_seg, N * up, N, up, has_bn, has_bn
    L.s_co, L.s_j = C_in, 1
    for i in range(n_seg):
        g = L.seg[i]
        g.C, g.tap, g.stride, g.s_ci, g.w_off = C_in, tap, stride, 1, 0
        g.src.T, g.src.up, g.src.ld, g.src.cup, g.src.c0 = T * stride, 1, C_in, C_in, 0
    return L


@pytest.mark.parametrize("shape", [dict(B=2, T=4096, C_in=3, N=64), dict(B=32, T=280, C_in=128, N=128),
                                   dict(B=32, T=140, C_in=256, N=256, n_seg=3, tap=-1),
                                   dict(B=4, T=35, C_in=128, N=256, up=4), dict(B=8, T=70, C_in=768, N=41, has_bn=0)])
def test_workspace_query_depends_on_the_shape_only(shape):
    lib = _lib.load()
    L1 = _layer(**shape)
    n1 = lib.fcn_train_deterministic_workspace_floats(C.byref(L1))
    assert n1 > 0
    L2 = _layer(**shape)                                 # other pointers, other source statistics: same size
    L2.W, L2.Y, L2.dW, L2.dA = 16, 32, 48, 64
    for i in range(L2.n_seg):
        L2.seg[i].src.raw, L2.seg[i].src.grad, L2.seg[i].src.count = 80, 96, 123.0
    assert lib.fcn_train_deterministic_workspace_floats(C.byref(L2)) == n1
    assert lib.fcn_train_deterministic_workspace_floats(None) == 0


def test_workspace_query_reads_only_whether_bias_is_set():
    """`bias` is structural: with BN it rules out the plain kernels (another split), so NULL or not matters; which
    address it holds does not."""
    lib = _lib.load()
    plain = dict(B=32, T=280, C_in=128, N=128)              # takes the plain kernels without a bias
    sizes = []
    for bias in (None, 16, 4096):
        L = _layer(**plain)
        L.bias = bias
        sizes.append(lib.fcn_train_deterministic_workspace_floats(C.byref(L)))
    assert sizes[1] == sizes[2] != sizes[0]
    L = _layer(B=8, T=70, C_in=768, N=41, has_bn=0)          # never plain: the bias changes nothing
    n0 = lib.fcn_train_deterministic_workspace_floats(C.byref(L))
    L.bias = 16
    assert lib.fcn_train_deterministic_workspace_floats(C.byref(L)) == n0


def test_loss_scratch_query():
    lib = _lib.load()
    assert lib.fcn_det_loss_deterministic_scratch_floats(1) == 16 + 13
    assert lib.fcn_det_loss_deterministic_scratch_floats(32 * 140) == 16 + 35 * 13
    assert lib.fcn_det_loss_deterministic_scratch_floats(0) == 0
    assert lib.fcn_det_loss_deterministic_scratch_floats((1 << 24) + 1) == 0


def test_null_and_small_workspace_are_rejected_before_any_launch():
    lib = _lib.load()
    L = _layer(B=2, T=64, C_in=16, N=32)
    L.W, L.Y, L.dW, L.dA, L.dsums, L.sums, L.gamma, L.beta = 16, 32, 48, 64, 80, 96, 112, 128
    for i in range(L.n_seg):
        L.seg[i].src.raw = 144
    need = lib.fcn_train_deterministic_workspace_floats(C.byref(L))
    for ws, n in ((None, need), (4096, need - 1)):
        assert lib.fcn_train_forward_deterministic(C.byref(L), ws, n, None) != 0
        assert b"workspace" in lib.fcn_last_error()
        assert lib.fcn_train_backward_deterministic(C.byref(L), 0, ws, n, None) != 0
        assert b"workspace" in lib.fcn_last_error()
