"""CPU: the frustum extractor's float64 restatement (oracle/frustum_extract.py) against the reference's own pickle
(tests/golden/frustum_extract.npz, oracle/make_golden_frustum_extract.py), the detection-line reader, the fixture's
edge cases, argument validation of the fcn_frustum_extract_* entries (on the host, before any CUDA call), the Python
wrappers' input checks and the kernels' register budget."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import ROOT
from toolchain import compile_cuda

GOLDEN = os.path.join(ROOT, "tests", "golden", "frustum_extract.npz")


def _scenes(part):
    from oracle import kitti_scan_synth as ks
    z = np.load(GOLDEN)
    return z, ks.fixture_scenes(z, part)


@pytest.mark.parametrize("part", ["exact", "real"])
def test_oracle_reproduces_the_reference_pickle(part):
    from frustum_convnet_b200.frustum_extract import read_rgb_detections
    from oracle import frustum_extract as ofx
    z, (scans, calibs, hw, lines) = _scenes(part)
    ids, types, probs, boxes = read_rgb_detections(lines)
    r_id, r_box, r_in, r_type, r_ang, r_prob, r_cal = ofx.extract(scans, calibs, hw, ids, types, probs, boxes,
                                                                  tuple(z[part + "_whitelist"]))
    assert r_id == z[part + "_ids"].tolist()
    assert r_type == z[part + "_types"].tolist()
    assert np.array(r_prob).tobytes() == z[part + "_probs"].tobytes()
    assert np.array(r_box).reshape(-1, 4).tobytes() == z[part + "_boxes"].tobytes()
    assert [len(p) for p in r_in] == z[part + "_counts"].tolist()
    assert np.concatenate(r_in).tobytes() == z[part + "_points"].tobytes()
    assert np.array(r_ang).tobytes() == z[part + "_angles"].tobytes()
    assert np.array([c["P2"] for c in r_cal]).tobytes() == z[part + "_P2"].tobytes()


def test_read_rgb_detections_equals_read_det_file():
    from frustum_convnet_b200.frustum_extract import read_rgb_detections
    z = np.load(GOLDEN)
    ids, types, probs, boxes = read_rgb_detections(str(s) for s in z["val_lines"])
    assert ids == z["val_ids"].tolist() and types == z["val_types"].tolist()
    assert np.array(probs).tobytes() == z["val_probs"].tobytes()
    assert np.array(boxes).tobytes() == z["val_boxes"].tobytes()
    assert len(set(types)) == 3
    with pytest.raises(ValueError):
        read_rgb_detections(["000001.png Van 0.5 1 2 3 4"])


def _rect(p):
    """exact_calib's velo -> rect, exact in float32 for the fixture's edge points."""
    return np.array([0.25 - p[0 + 1], -0.5 - p[2], p[0] - 0.25, p[3]], dtype=np.float32)


def test_exact_part_covers_the_edges():
    from oracle import kitti_scan_synth as ks
    z = np.load(GOLDEN)
    lines = [str(s) for s in z["exact_lines"]]
    kept_lines = [lines[i] for i in (0, 1, 2, 4, 5, 9, 10)]         # see kitti_scan_synth.exact_scene
    assert z["exact_boxes"].tolist() == [
        [400, 150, 440, 190], [0, 195, 30, 215], [500, 200, 540, 205], [1200, 100, 1241, 140], [620, 150, 640, 175],
        [900, 150, 960, 200], [930, 170, 1000, 230]]
    assert z["exact_ids"].tolist() == [ks.det_id(ln) for ln in kept_lines] == [3, 3, 5, 3, 3, 5, 5]
    off = np.concatenate([[0], np.cumsum(z["exact_counts"])])
    pts = [z["exact_points"][off[k]:off[k + 1]] for k in range(len(off) - 1)]
    has = lambda k, p: any(np.array_equal(q, _rect(p)) for q in pts[k])
    ep = ks.exact_point
    assert has(0, ep(400, 170)) and not has(0, ep(440, 170))            # u on xmin / xmax
    assert has(0, ep(420, 150)) and not has(0, ep(420, 190))            # v on ymin / ymax
    assert has(1, ep(0, 200))                                           # u = 0, box clipped from xmin = -20
    assert not any(has(k, ep(ks.W, 200)) for k in range(len(pts)))      # u = W
    assert has(3, ep(1240.5, 120)) and not has(3, ep(1241.5, 120))      # box clipped to W - 1
    two = np.array([2.0, 0.25, -0.5, 0.25], np.float32)
    after = two.copy()
    after[0] = np.nextafter(np.float32(2.0), np.float32(3))
    assert has(4, after) and not has(4, two)                           # x_velo = 2.0f dropped, next float kept
    assert not np.isnan(z["exact_points"]).any()
    overlap = {q.tobytes() for q in pts[5]} & {q.tobytes() for q in pts[6]}
    assert overlap                                                      # overlapping boxes share points


def test_c_entries_validate_without_gpu():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    A = _lib.FrustumExtractArgs
    assert lib.fcn_frustum_extract_count(None, None) == -1
    assert b"NULL" in lib.fcn_last_error()
    assert lib.fcn_frustum_extract_workspace_bytes(None) == -1
    a = A()
    assert lib.fcn_frustum_extract_count(ctypes.byref(a), None) == 0          # zero frames: nothing to do
    assert lib.fcn_frustum_extract_write(ctypes.byref(a), None) == 0
    assert lib.fcn_frustum_extract_workspace_bytes(ctypes.byref(a)) == 0
    a.num_frames, a.num_points, a.num_dets = 2, 10, 0
    assert lib.fcn_frustum_extract_count(ctypes.byref(a), None) == 0          # zero detections
    a.num_dets = -1
    assert lib.fcn_frustum_extract_count(ctypes.byref(a), None) == -1
    assert b"negative" in lib.fcn_last_error()
    a.num_dets, a.num_frames = 3, 70000
    assert lib.fcn_frustum_extract_count(ctypes.byref(a), None) == -1
    a.num_frames = 2
    assert lib.fcn_frustum_extract_count(ctypes.byref(a), None) == -1      # NULL host offsets
    so = np.array([0, 4, 10], dtype=np.int32)
    a.host_scan_offsets = so.ctypes.data
    assert lib.fcn_frustum_extract_count(ctypes.byref(a), None) == -1      # NULL device pointers
    assert b"NULL" in lib.fcn_last_error()
    buf = np.zeros(64, dtype=np.float32)
    base = buf.ctypes.data + (-buf.ctypes.data) % 16
    a.scans, a.scan_offsets, a.frames, a.boxes, a.det_frame = base + 4, base, base, base, base
    assert lib.fcn_frustum_extract_count(ctypes.byref(a), None) == -1
    assert b"aligned" in lib.fcn_last_error()
    a.scans = base
    for bad in ([1, 4, 10], [0, 5, 4], [0, 4, 11]):
        so[:] = bad
        assert lib.fcn_frustum_extract_count(ctypes.byref(a), None) == -1
        assert b"offsets" in lib.fcn_last_error()
    so[:] = [0, 4, 10]
    assert lib.fcn_frustum_extract_count(ctypes.byref(a), None) == -1      # NULL workspace / info
    assert b"workspace" in lib.fcn_last_error()
    assert lib.fcn_frustum_extract_write(ctypes.byref(a), None) == -1


def test_wrappers_reject_cpu_tensors_and_mismatched_lists():
    from frustum_convnet_b200.frustum_extract import FrustumExtractor
    from frustum_convnet_b200.input_builder import FrustumBatchBuilder
    with pytest.raises(RuntimeError):
        FrustumExtractor(device="cpu")
    ex = FrustumExtractor(device="cuda")
    cal = {"P2": np.zeros(12), "Tr_velo_to_cam": np.zeros(12), "R0_rect": np.eye(3)}
    box = [np.array([0.0, 0, 10, 10])]
    with pytest.raises(ValueError):
        ex.extract({1: np.zeros((4, 4), np.float32)}, {1: cal}, {1: (10, 10)}, [1], ["Car"], [0.5, 0.6], box)
    with pytest.raises(ValueError):
        ex.extract({1: np.zeros((4, 4), np.float32)}, {1: cal}, {1: (10, 10)}, [1, 1], ["Car"], [0.5], box)
    with pytest.raises(RuntimeError):
        ex.extract({1: torch.zeros(4, 4)}, {1: cal}, {1: (10, 10)}, [1], ["Car"], [0.5], box)
    with pytest.raises(ValueError):
        ex.extract({1: np.zeros((4, 3), np.float32)}, {1: cal}, {1: (10, 10)}, [1], ["Car"], [0.5], box)
    fb = FrustumBatchBuilder([0.25, 0.5, 1.0, 2.0], 70.0, 1024)
    with pytest.raises(RuntimeError):
        fb.set_frustums_device(torch.zeros(5, 4), torch.tensor([0, 5], dtype=torch.int32),
                               torch.zeros(1, dtype=torch.float64), torch.zeros(1, 4, dtype=torch.float64),
                               torch.zeros(1, 12, dtype=torch.float64))


def test_detection_extraction_kernels_compile_without_spills():
    """The detection extractor's own kernels (csrc/frustum_extract.cu) and the stage it shares with the other
    extractors (csrc/frustum_fov.cu, the family's only CUB device scans) compile for sm_90a without spills."""
    reports = {src: compile_cuda(src + ".cu").kernels for src in ("frustum_extract", "frustum_fov")}

    def named(src, *parts):
        return sorted(p for p in parts if any(p in k for k in reports[src]))

    own = ("fx_count_kernel", "fx_write_kernel")
    shared = ("fov_flag_kernel", "fov_compact_kernelILb0", "fov_compact_kernelILb1", "job_info_kernel")
    assert named("frustum_extract", *own) == sorted(own) and len(reports["frustum_extract"]) == 2, \
        sorted(reports["frustum_extract"])
    assert named("frustum_fov", *shared) == sorted(shared), sorted(reports["frustum_fov"])
    assert any("DeviceScanKernel" in k for k in reports["frustum_fov"]), sorted(reports["frustum_fov"])
    for src in reports:
        for name, k in reports[src].items():
            assert (k.spill_stores, k.spill_loads) == (0, 0), name + "\n" + k.report
