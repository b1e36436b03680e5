"""CPU: the frame refinement entries (C ABI section (22)) without a GPU: their argument checks, the section-width rule
against the refinement provider's own arange, the ptxas usage of the new kernels, and the SASS of the batch kernel
that became a template instantiation."""
import ctypes as C
import hashlib

import numpy as np
import pytest

from toolchain import compile_cuda, nvcc_release

# cuobjdump -sass of build_train_inputs_kernel before it became the <false> instantiation (CUDA 12.9, sm_90a, the
# build's flags): the fixed-width path must leave the batch-maximum path's instructions byte for byte as they were
PARENT_SASS = {"12.9": "c2db9bebe2b77c219111f1dbc6ce6330c4ac22c5caa76e0a495c37befd218dfc"}


def _args():
    from frustum_convnet_b200 import _lib
    a = _lib.FrameRefineArgs()
    a.num_frames, a.scan_capacity, a.job_capacity, a.out_capacity, a.num_rows, a.num_scales = 1, 16, 4, 16, 8, 4
    for s, (st, w) in enumerate(zip((0.1, 0.2, 0.4, 0.8), (48, 24, 12, 6))):
        a.stride[s], a.widths[s] = st, w
    return a


def test_entry_argument_checks_without_gpu():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    assert lib.fcn_frame_refine_extract(None, None) == -1
    assert lib.fcn_frame_refine_extract_workspace_bytes(None) == -1
    for field in ("num_frames", "scan_capacity", "job_capacity", "out_capacity", "num_rows"):
        a = _args()
        setattr(a, field, 0)
        assert lib.fcn_frame_refine_extract_workspace_bytes(C.byref(a)) == -1, field
        assert b">= 1" in lib.fcn_last_error(), field
    a = _args()
    a.widths[2] = 0
    assert lib.fcn_frame_refine_extract_workspace_bytes(C.byref(a)) == -1
    assert b"widths" in lib.fcn_last_error()
    a = _args()
    a.num_scales = 9
    assert lib.fcn_frame_refine_extract_workspace_bytes(C.byref(a)) == -1
    a = _args()
    a.out_capacity = 1 << 24
    assert lib.fcn_frame_refine_extract_workspace_bytes(C.byref(a)) == -1
    assert b"too large" in lib.fcn_last_error()
    a = _args()
    assert lib.fcn_frame_refine_extract(C.byref(a), None) == -1
    assert b"NULL input" in lib.fcn_last_error()
    for name in ("scans", "scan_counts", "frames", "rows", "seg_offsets", "keep_count", "seg_class", "status"):
        setattr(a, name, 256)
    assert lib.fcn_frame_refine_extract(C.byref(a), None) == -1
    assert b"NULL output" in lib.fcn_last_error()
    # the resampling of the refinement batch: N outside 1..2048 is refused
    r = _lib.ResampleArgs()
    for N in (0, 2049):
        r.B, r.N = 1, N
        assert lib.fcn_resample_choice(C.byref(r), None) == -1


def test_fixed_batch_argument_checks_without_gpu():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    w = (C.c_int32 * 4)(48, 24, 12, 6)
    assert lib.fcn_build_train_inputs_fixed(None, w, None) == -1
    t = _lib.TrainInputArgs()
    t.kind, t.labels, t.rtc, t.B, t.N, t.num_scales, t.num_classes, t.num_frustums = _lib.TRAIN_REFINE, 0, 1, 0, 512, \
        4, 3, 1
    for s in range(4):
        t.stride[s], t.centers[s] = 0.1 * 2 ** s, 256
    assert lib.fcn_build_train_inputs_fixed(C.byref(t), None, None) == -1
    assert b"NULL widths" in lib.fcn_last_error()
    bad = (C.c_int32 * 4)(48, 0, 12, 6)
    assert lib.fcn_build_train_inputs_fixed(C.byref(t), bad, None) == -1
    assert b"widths" in lib.fcn_last_error()
    assert lib.fcn_build_train_inputs_fixed(C.byref(t), w, None) == 0          # B = 0: nothing to do
    t.B = 2
    assert lib.fcn_build_train_inputs_fixed(C.byref(t), w, None) == -1
    assert b"NULL pointer" in lib.fcn_last_error()
    t.N = 0
    assert lib.fcn_build_train_inputs_fixed(C.byref(t), w, None) == -1


@pytest.mark.parametrize("width", [0.05, 0.1, 0.4, 1.0, 1.92, 2.0, 4.8, 4.80000001, 7.3])
def test_section_widths_follow_the_refine_ref_line(width):
    """W[s] of max_width w is the T[s] refine_ref_line gives a predicted box of width w."""
    from frustum_convnet_b200.frame_detect import section_widths
    from frustum_convnet_b200.refine_extract import REFINE_STRIDES, compute_box_3d_obj_array
    from frustum_convnet_b200.train_inputs import refine_ref_line
    for ry in (0.0, 0.7, -2.9):
        a = np.array([1.5, 1.2, 20.0, 4.2, width, 1.6, ry])
        Ts = refine_ref_line(compute_box_3d_obj_array(a), a[3:6], ry, REFINE_STRIDES)[4]
        assert section_widths(width, REFINE_STRIDES) == Ts, (width, ry)


@pytest.mark.parametrize("src,kernels,max_regs", [
    ("frame_refine.cu", ["fr_plan_kernel", "fr_slots_kernel"], 64),
    ("train_inputs.cu", ["build_train_inputs_kernelILb1EE"], 255),
])
def test_new_kernels_do_not_spill(src, kernels, max_regs):
    seen = set()
    for name, k in compile_cuda(src).kernels.items():
        for want in kernels:
            if want in name:
                seen.add(want)
                assert (k.spill_stores, k.spill_loads) == (0, 0), (name, k.report)
                assert k.registers <= max_regs, name
    assert seen == set(kernels)


def test_batch_kernel_sass_is_the_parents():
    version = nvcc_release()
    if version not in PARENT_SASS:
        pytest.skip("the parent's SASS digest was taken with CUDA %s" % sorted(PARENT_SASS))
    bodies = compile_cuda("train_inputs.cu").sass()
    false = [b for n, b in bodies.items() if "build_train_inputs_kernelILb0E" in n]
    assert len(false) == 1 and any("build_train_inputs_kernelILb1E" in n for n in bodies)
    assert hashlib.sha256(false[0].encode()).hexdigest() == PARENT_SASS[version]
