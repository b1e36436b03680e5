"""GPU: every two-phase entry family (detect, kitti_eval, sunrgbd_eval, frustum_extract, refine_extract, gt_extract)
checks the caller's workspace against its fcn_*_workspace_bytes() size.  Each family runs through its public class on
a small valid input; every entry call that takes a workspace is first replayed one byte short, which must be refused
with the size function's name before any device work, and then runs with exactly the queried size."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ENTRIES = {
    "det": ("fcn_det_prepare", "fcn_det_select"),
    "kitti_eval": ("fcn_kitti_eval_overlaps", "fcn_kitti_eval_thresholds", "fcn_kitti_eval_statistics"),
    "sunrgbd_eval": ("fcn_sunrgbd_eval_match", "fcn_sunrgbd_eval_curves"),
    "frustum_extract": ("fcn_frustum_extract_count", "fcn_frustum_extract_write"),
    "refine_extract": ("fcn_refine_extract_count", "fcn_refine_extract_write"),
    "gt_extract": ("fcn_gt_extract_count", "fcn_gt_extract_write"),
}


def _detect():
    from test_gpu_kitti_eval import _collector_output
    assert _collector_output()


def _kitti_eval():
    from frustum_convnet_b200.kitti_eval import KittiEvaluator, KittiGroundTruth
    from oracle import kitti_synth as ks
    labels, results = ks.make_set(101, 8, check_margins=True, n_obj=4, det_rate=0.8)
    gt = KittiGroundTruth(list(range(8)), [ks.parse_label_lines(l) for l in labels])
    KittiEvaluator(gt).evaluate_records([ks.parse_result_lines(r) for r in results])


def _sunrgbd_eval():
    from frustum_convnet_b200.sunrgbd_eval import SunrgbdEvaluator
    from oracle import sunrgbd_synth as ss
    from test_gpu_sunrgbd_eval import _gt
    classes = ("bed", "table", "chair")
    rows, ids, det = ss.make_set(31, 12, classes, fp_rate=2.0)
    SunrgbdEvaluator(_gt(rows, ids, classes)).evaluate(det)


def _frustum_extract():
    from oracle import kitti_scan_synth as ks
    from test_gpu_frustum_extract import GOLDEN, _extract
    z = np.load(GOLDEN)
    scans, calibs, hw, lines = ks.fixture_scenes(z, "real")
    assert len(_extract(scans, calibs, hw, lines, tuple(z["real_whitelist"])))


def _refine_extract():
    from oracle import kitti_refine_synth as krs
    from test_gpu_refine_extract import GOLDEN, _run
    z = np.load(GOLDEN)
    scans, calibs, hws, labels, results = krs.fixture_scenes(z)
    assert len(_run("matched", scans, calibs, hws, z["frame_ids"].tolist(), labels, results))


def _gt_extract():
    from test_gpu_gt_extract import _run, scenes
    z, scans, calibs, hws, labels, dets = scenes()
    assert len(_run("car_matched", scans, calibs, hws, z["frame_ids"].tolist(), labels, dets,
                    np.random.RandomState(1)))


RUN = {"det": _detect, "kitti_eval": _kitti_eval, "sunrgbd_eval": _sunrgbd_eval, "frustum_extract": _frustum_extract,
       "refine_extract": _refine_extract, "gt_extract": _gt_extract}


@pytest.mark.parametrize("family", sorted(ENTRIES))
def test_one_byte_short_is_refused_and_the_queried_size_runs(family, monkeypatch):
    from frustum_convnet_b200 import _lib
    lib, real_call, seen = _lib.load(), _lib.call, []

    def call(name, *args):
        if name in ENTRIES[family]:
            a = args[0]._obj
            if family == "det":
                n = lib.fcn_det_workspace_bytes(a.capacity, a.num_segments)
            else:
                n = getattr(lib, "fcn_%s_workspace_bytes" % family)(ctypes.byref(a))
            assert n > 0 and a.workspace_bytes == n, (name, n, a.workspace_bytes)
            a.workspace_bytes = n - 1
            assert getattr(lib, name)(*args) == -1, name
            err = lib.fcn_last_error()
            assert b"workspace smaller than fcn_%s_workspace_bytes()" % family.encode() in err, err
            a.workspace_bytes = n
            seen.append(name)
        real_call(name, *args)                   # raises unless the entry returns 0

    monkeypatch.setattr(_lib, "call", call)
    RUN[family]()
    assert set(seen) == set(ENTRIES[family]), seen
