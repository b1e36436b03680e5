"""CPU: the SUN-RGBD frame entries (C ABI section (23)) without a GPU: their argument checks, the ptxas usage of the
new kernels, and the SASS of every existing kernel the frame path launches, which must stay as it was."""
import ctypes as C
import hashlib

import pytest

from toolchain import compile_cuda, nvcc_release

# cuobjdump -sass digests (CUDA 12.9, sm_90a, the build's flags) of the kernels the SUN-RGBD frame path reuses, taken
# before it was added: section (18)'s sx_* (csrc/sunrgbd_extract.cu now shares its box test with the frame path), the
# resampling, the batch builder and the collector
PARENT_SASS = {"12.9": {
    ("sunrgbd_extract.cu", "_ZN3fcn15sx_write_kernelILb0EEEvixPKiPK10fcn_gt_jobPK14fcn_refine_boxPKfPKdSC_S2_S2_S2_S2_S2_PKxPfPhPi"):
        "4af307c6054099d1ef9fce78cffbe64b4ebdfece8064623c1e293facaa803f3d",
    ("sunrgbd_extract.cu", "_ZN3fcn15sx_write_kernelILb1EEEvixPKiPK10fcn_gt_jobPK14fcn_refine_boxPKfPKdSC_S2_S2_S2_S2_S2_PKxPfPhPi"):
        "6a0d623924c6ac79198f02084f873cf4233d331ec5fff2b8d7d95c841597787c",
    ("sunrgbd_extract.cu", "_ZN3fcn16sx_select_kernelILb0EEEviPKiPK10fcn_gt_jobPK14fcn_refine_boxPKfPKdSC_PiS2_S2_S2_SD_PxSD_"):
        "2f091891014c1c48b52aa7493eb1699d33c500ecf61b575861aeb58a5691b0d3",
    ("sunrgbd_extract.cu", "_ZN3fcn16sx_select_kernelILb1EEEviPKiPK10fcn_gt_jobPK14fcn_refine_boxPKfPKdSC_PiS2_S2_S2_SD_PxSD_"):
        "e1bc7ceb48f95e20333ee929afc6a2fcd4e169b73585d806024078e218c8df7f",
    ("sunrgbd_extract.cu", "_ZN3fcn15sx_count_kernelILb0EEEviiiPKiPK10fcn_gt_jobPK14fcn_refine_boxPKfPKdSC_PiSD_SD_"):
        "01cbaed61ea751c3e397cf7c28caa863311cdde2ed3d924315322d9404d19a19",
    ("sunrgbd_extract.cu", "_ZN3fcn15sx_count_kernelILb1EEEviiiPKiPK10fcn_gt_jobPK14fcn_refine_boxPKfPKdSC_PiSD_SD_"):
        "9138cb251dfa8e297664ce6c37d77023333e5ba7977fca06e987b8c2b09a3607",
    ("sunrgbd_extract.cu", "_ZN3fcn17sx_project_kernelEPKfPKiPK17fcn_sunrgbd_framePdS7_"):
        "58b8d008b3f8e6f74647c0d9f4384b54745487c75c4bcb4cd4210951f7e5f550",
    ("resample.cu", "_ZN3fcn22resample_choice_kernelE17fcn_resample_args"):
        "6b28634d8a50c22952097b71a6c4d4a8bbab6432605495a897d4b8f238b0f175",
    ("train_inputs.cu", "_ZN3fcn25build_train_inputs_kernelILb1EEEv20fcn_train_input_argsNS_6WidthsE"):
        "7731d9123a0e8144b0974d78f13b65bdafd28727dd8c2c43a0fac3c9be673f4c",
    ("train_inputs.cu", "_ZN3fcn25build_train_inputs_kernelILb0EEEv20fcn_train_input_argsNS_6WidthsE"):
        "c2db9bebe2b77c219111f1dbc6ce6330c4ac22c5caa76e0a495c37befd218dfc",
    ("detect.cu", "_ZN3fcn15det_rows_kernelILb1EEEviiiPK14fcn_det_recordPKiS5_S5_S5_PKfPfS5_"):
        "db9a39bb8282495fce9272fcaca73d968b1b2087f79a02acdabd40239f68dc87",
    ("detect.cu", "_ZN3fcn15det_rank_kernelILb1EEEviPK14fcn_det_recordPKiS5_PiPfS7_S5_"):
        "b3070bc5f0534dec9f6bd4b1e758a79c2fb3a99876c4c246c087d633864b7e8f",
    ("detect.cu", "_ZN3fcn19det_overflow_kernelEiPKiPi"):
        "415506f771ee48954eab6e1d3bf829e87c516c6b4fde797372001ca769e1840d",
    ("detect.cu", "_ZN3fcn15det_rows_kernelILb0EEEviiiPK14fcn_det_recordPKiS5_S5_S5_PKfPfS5_"):
        "cb8018a1e80d4a8557842fdc8a08fa96fa4c1d54955a7d1e8b4ff717ebdf35a4",
    ("detect.cu", "_ZN3fcn15det_rank_kernelILb0EEEviPK14fcn_det_recordPKiS5_PiPfS7_S5_"):
        "4026c767fd3459abc59776aaf1f86c116fbdc8272acb05b6b5c3a34a7fea0afc",
    ("detect.cu", "_ZN3fcn21det_candidates_kernelILb1EEEv22fcn_det_candidate_argsPKi"):
        "7cdb1ae972fbb0a33c496b0ddb6de3514a2a0d2a0ad135899e913fdb9a4c66b3",
    ("detect.cu", "_ZN3fcn21det_candidates_kernelILb0EEEv22fcn_det_candidate_argsPKi"):
        "39b5b05064ced116579b8e406709611e22efd21c3d81c0ab3c8314fed827536f",
    ("detect.cu", "_ZN3fcn15det_scan_kernelEiiiPKiPKxPKjPjPiS7_"):
        "487121eee9fc3eea3b950955f1395fc6378e1daa9c7dc68795adea992cfb6dfd",
    ("detect.cu", "_ZN3fcn16det_pairs_kernelEifPKiPKxS3_PKfS5_Pj"):
        "d3a646cb2c1f60964a6648a4066b85d7760674318bd752c7a6f34a122898969d",
    ("detect.cu", "_ZN3fcn15det_info_kernelEiPKiPKxS3_Px"):
        "cafa881be71812e2ba11b7146ee75054e648718ee92670bbb513ab5005d83bf2",
    ("detect.cu", "_ZN3fcn20det_seg_sizes_kernelEiiPKiPxS2_"):
        "1121694b8fac6a6678cc50aa5d70c533600521c512d177da5884e22d62ba36c7",
    ("detect.cu", "_ZN3fcn24det_gather_sorted_kernelEiPKiiPK14fcn_det_recordS1_PS2_PyPi"):
        "49a080c9fe183e0962b9cd90171c9470cdc1f993f8910ae1dce6eaf1caefdf0b",
    ("detect.cu", "_ZN3fcn15det_keys_kernelEiPKiPK14fcn_det_recordPyPiS6_"):
        "ce6fd2319cfca6277626fa657a6bd2ffb86978d2eaf138af9e49986a6de07c62",
}}


def _args():
    from frustum_convnet_b200 import _lib
    a = _lib.SunrgbdFrameExtractArgs()
    a.num_frames, a.point_capacity, a.det_capacity, a.out_capacity = 2, 1024, 8, 4096
    a.class_mask, a.num_scales, a.max_depth = 0x3FF, 5, 8.0
    for s, st in enumerate((0.1, 0.2, 0.4, 0.8, 1.6)):
        a.stride[s] = st
    return a


def test_entry_argument_checks_without_gpu():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    assert lib.fcn_sunrgbd_frame_extract(None, None) == -1
    assert lib.fcn_sunrgbd_frame_extract_workspace_bytes(None) == -1
    for field in ("num_frames", "point_capacity", "det_capacity", "out_capacity"):
        a = _args()
        setattr(a, field, 0)
        assert lib.fcn_sunrgbd_frame_extract_workspace_bytes(C.byref(a)) == -1, field
        assert b">= 1" in lib.fcn_last_error(), field
    a = _args()
    a.det_capacity = 65
    assert lib.fcn_sunrgbd_frame_extract_workspace_bytes(C.byref(a)) == -1
    assert b"<= 64" in lib.fcn_last_error()
    for field, value in (("point_capacity", 1 << 24), ("out_capacity", 1 << 24), ("num_frames", 65536)):
        a = _args()
        setattr(a, field, value)
        assert lib.fcn_sunrgbd_frame_extract_workspace_bytes(C.byref(a)) == -1, field
        assert b"too large" in lib.fcn_last_error(), field
    a = _args()
    a.num_frames, a.det_capacity, a.point_capacity = 4096, 64, 1 << 13          # F * D * P = 2^31
    assert lib.fcn_sunrgbd_frame_extract_workspace_bytes(C.byref(a)) == -1
    a = _args()
    a.class_mask = 1 << 10
    assert lib.fcn_sunrgbd_frame_extract_workspace_bytes(C.byref(a)) == -1
    assert b"class_mask" in lib.fcn_last_error()
    for field, value in (("num_scales", 0), ("num_scales", 9), ("max_depth", 0.0), ("max_depth", float("inf"))):
        a = _args()
        setattr(a, field, value)
        assert lib.fcn_sunrgbd_frame_extract_workspace_bytes(C.byref(a)) == -1, (field, value)
    a = _args()
    a.stride[3] = -0.4
    assert lib.fcn_sunrgbd_frame_extract_workspace_bytes(C.byref(a)) == -1
    assert b"strides" in lib.fcn_last_error()
    a = _args()
    assert lib.fcn_sunrgbd_frame_extract(C.byref(a), None) == -1
    assert b"NULL input" in lib.fcn_last_error()
    for name in ("clouds", "cloud_counts", "frames", "boxes", "det_class", "det_prob", "det_counts", "call", "status"):
        setattr(a, name, 256)
    assert lib.fcn_sunrgbd_frame_extract(C.byref(a), None) == -1
    assert b"NULL output" in lib.fcn_last_error()
    for name in ("points", "xyz", "offsets", "det_index", "valid", "cls_index", "seg", "seg_class", "rgb_prob", "box2d",
                 "cap_choice", "records"):
        setattr(a, name, 256)
    a.clouds = 258
    assert lib.fcn_sunrgbd_frame_extract(C.byref(a), None) == -1
    assert b"aligned" in lib.fcn_last_error()
    a.clouds = 256
    assert lib.fcn_sunrgbd_frame_extract(C.byref(a), None) == -1                # no workspace
    assert b"workspace" in lib.fcn_last_error()


def test_detector_argument_checks_without_gpu():
    from frustum_convnet_b200.frame_detect import SunrgbdFrameDetector
    with pytest.raises(ValueError, match="unknown types"):
        SunrgbdFrameDetector(None, type_whitelist=("Car",))
    with pytest.raises((RuntimeError, ValueError)):
        SunrgbdFrameDetector(None, device="cpu")


@pytest.mark.parametrize("kernel,max_regs", [
    ("sf_setup_kernel", 32), ("sf_project_kernel", 64), ("sf_points_kernelILb0E", 64),
    ("sf_points_kernelILb1E", 64), ("sf_scan_kernel", 32), ("sf_slots_kernel", 64), ("sf_sort_kernel", 64),
    ("sf_records_kernel", 64),
])
def test_new_kernels_do_not_spill(kernel, max_regs):
    found = [(n, k) for n, k in compile_cuda("sunrgbd_frame.cu").kernels.items() if kernel in n]
    assert len(found) == 1
    name, k = found[0]
    assert (k.spill_stores, k.spill_loads) == (0, 0), (name, k.report)
    assert k.registers <= max_regs, (name, k.registers)


def test_reused_kernels_sass_is_the_parents():
    version = nvcc_release()
    if version not in PARENT_SASS:
        pytest.skip("the parent's SASS digests were taken with CUDA %s" % sorted(PARENT_SASS))
    for (src, name), digest in PARENT_SASS[version].items():
        body = compile_cuda(src).sass().get(name)
        assert body is not None, name
        assert hashlib.sha256(body.encode()).hexdigest() == digest, name
