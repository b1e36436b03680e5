"""CPU: the SUN-RGBD evaluator's numpy restatement (oracle/sunrgbd_eval.py) against the reference's own eval_det_cls
output (tests/golden/sunrgbd_eval.npz, oracle/make_golden_sunrgbd_eval.py), the ground-truth file parser and
conversion, the corner construction, the stable tie rule, the no-detection divergence, and argument validation of the
fcn_sunrgbd_eval_* entries (done on the host, before any CUDA call)."""
import ctypes
import os

import numpy as np
import pytest

from conftest import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden", "sunrgbd_eval.npz")
RUNS = ("synth", "real")


def fixture(run):
    """-> (classes, gt rows {class: (n, 10)}, gt ids {class: (n,)}, det_results {idx: {class: (n, 12)}}, pred_all
    {class: {idx: [(corners, score)]}} (the reference's corners), expected {class: (rec, prec, ap)}, lines)."""
    z = np.load(GOLDEN)
    classes = [str(c) for c in z[run + "_classes"]]
    cnt = np.concatenate([[0], np.cumsum(z[run + "_gt_class_counts"])])
    rows = {c: z[run + "_gt_rows"][cnt[i]:cnt[i + 1]] for i, c in enumerate(classes)}
    ids = {c: z[run + "_gt_ids"][cnt[i]:cnt[i + 1]] for i, c in enumerate(classes)}
    det = {}
    for r, i, c in zip(z[run + "_det_rows"], z[run + "_det_img"], z[run + "_det_cls"]):
        det.setdefault(int(i), {}).setdefault(str(c), []).append(r)
    det = {i: {c: np.stack(v) for c, v in by.items()} for i, by in det.items()}
    pred_all, k = {}, 0
    cor, sc = z[run + "_ref_corners"], z[run + "_ref_scores"]
    for c in classes:                                   # gather order: class, then image in dict order, then row
        for i, by in det.items():
            for _ in range(len(by.get(c, []))):
                pred_all.setdefault(c, {}).setdefault(i, []).append((cor[k], sc[k]))
                k += 1
    assert k == len(cor)
    nd = np.concatenate([[0], np.cumsum(z[run + "_nd"])])
    want = {c: (z[run + "_rec"][nd[j]:nd[j + 1]], z[run + "_prec"][nd[j]:nd[j + 1]], float(z[run + "_ap"][j]))
            for j, c in enumerate(classes)}
    return classes, rows, ids, det, pred_all, want, [str(s) for s in z[run + "_lines"]]


def write_gt_dir(tmp, run):
    z = np.load(GOLDEN)
    for c, dat, txt in zip(z[run + "_classes"], z[run + "_gt_dat"], z[run + "_gt_ids_txt"]):
        (tmp / ("%s_gt_boxes.dat" % c)).write_text(str(dat))
        (tmp / ("%s_gt_imgids.txt" % c)).write_text(str(txt))
    return str(tmp)


@pytest.mark.parametrize("run", RUNS)
def test_oracle_matches_the_reference_eval_det_cls(run):
    from oracle import sunrgbd_eval as ose
    classes, rows, ids, det, pred_all, want, lines = fixture(run)
    gt = ose.gt_from_rows(rows, ids)
    for got in (ose.evaluate(ose.gather_rows(det, classes), gt), ose.evaluate(ose.gather_corners(pred_all, classes), gt)):
        for c in classes:
            rec, prec, ap = want[c]
            assert np.array_equal(got["rec"][c], rec) and np.array_equal(got["prec"][c], prec), c
            assert abs(got["ap"][c] - ap) <= 1e-15, c
        assert got["lines"] == lines
    if run == "synth":
        assert len(want["chair"][0]) == 0 and want["chair"][2] == 0.0       # ground truth, no detection: AP 0


@pytest.mark.parametrize("run", RUNS)
def test_gt_parser_and_conversion(run, tmp_path):
    from frustum_convnet_b200 import sunrgbd_eval as se
    from oracle import sunrgbd_eval as ose
    classes, rows, ids, *_ = fixture(run)
    d = write_gt_dir(tmp_path, run)
    n_cw = n_ccw = 0
    for c in classes:
        boxes, img = se.read_gt_files(d, c)
        assert np.array_equal(boxes, rows[c]) and np.array_equal(img, ids[c])
        cor = se.gt_corners(boxes)
        assert np.array_equal(cor, np.stack([ose.gt_box_corners(r) for r in boxes]))
        xy = boxes[:, :8].reshape(-1, 4, 2)
        twice = (xy[..., 0] * np.roll(xy[..., 1], 1, 1) - xy[..., 1] * np.roll(xy[..., 0], 1, 1)).sum(1)
        n_cw += int((twice > 0).sum())
        n_ccw += int((twice < 0).sum())
        # the converted ring (x, z of corners 6, 7, 4, 5) is clockwise-positive and the height positive
        ring = cor[:, [6, 7, 4, 5]][..., [0, 2]]
        area = -(ring[..., 0] * np.roll(ring[..., 1], -1, 1) - np.roll(ring[..., 0], -1, 1) * ring[..., 1]).sum(1)
        assert (area > 0).all() and (cor[:, 0, 1] > cor[:, 4, 1]).all()
    if run == "synth":
        assert n_cw > 100 and n_ccw > 100


def test_one_row_class_and_bad_ids(tmp_path):
    from frustum_convnet_b200 import sunrgbd_eval as se
    (tmp_path / "bed_gt_boxes.dat").write_text("1 0 1 1 0 1 0 0 -1.5 0.5\n")
    (tmp_path / "bed_gt_imgids.txt").write_text("42\n")
    boxes, ids = se.read_gt_files(str(tmp_path), "bed")
    assert boxes.shape == (1, 10) and ids.tolist() == [42]
    cor = se.gt_corners(boxes)
    assert cor.shape == (1, 8, 3)
    assert np.array_equal(cor[0, :4, 1], [1.5] * 4) and np.array_equal(cor[0, 4:, 1], [-0.5] * 4)
    (tmp_path / "bed_gt_imgids.txt").write_text("42.5\n")
    with pytest.raises(ValueError):
        se.read_gt_files(str(tmp_path), "bed")
    (tmp_path / "bed_gt_imgids.txt").write_text("42 43\n")
    with pytest.raises(ValueError):
        se.read_gt_files(str(tmp_path), "bed")
    assert se.image_key(7.0) == 7 and se.image_key(np.int64(9)) == 9


@pytest.mark.parametrize("run", RUNS)
def test_detection_corners_follow_compute_box_3d(run):
    from frustum_convnet_b200 import sunrgbd_eval as se
    from oracle import sunrgbd_eval as ose
    classes, _, _, det, pred_all, *_ = fixture(run)
    rows = np.concatenate([by[c] for c in classes for by in det.values() if c in by])
    ref = np.stack([b for c in classes for lst in pred_all.get(c, {}).values() for b, _ in lst])
    mine = se.det_corners(rows)
    np.testing.assert_allclose(mine, ref, rtol=0, atol=1e-12)
    np.testing.assert_allclose(mine, np.stack([ose.det_box_corners(r) for r in rows]), rtol=0, atol=1e-12)


def _tie_case():
    """One ground truth G in image 1; detection A on G in image 1, detection B in image 2 (no ground truth), equal
    scores (one of them -0.0 against 0.0 in the second class)."""
    from oracle import sunrgbd_eval as ose
    from oracle import sunrgbd_synth as ss
    p = np.array([0.0, 0.5, 4.0, 2.0, 1.0, 1.0, 0.3])
    g = ose.gt_box_corners(ss.gt_row(p, False))
    a = ss.det_row(p, 0.7)
    b = ss.det_row(p + [3, 0, 0, 0, 0, 0, 0], 0.7)
    return g, a, b


def test_ties_rank_by_gather_order():
    from oracle import sunrgbd_eval as ose
    g, a, b = _tie_case()
    gt = {"bed": {1: [g]}}
    first = ose.evaluate(ose.gather_rows({1: {"bed": a[None]}, 2: {"bed": b[None]}}, ["bed"]), gt)
    second = ose.evaluate(ose.gather_rows({2: {"bed": b[None]}, 1: {"bed": a[None]}}, ["bed"]), gt)
    assert first["prec"]["bed"].tolist() == [1.0, 0.5] and first["ap"]["bed"] == 1.0
    assert second["prec"]["bed"].tolist() == [0.0, 0.5] and second["ap"]["bed"] == 0.5
    a0, b0 = a.copy(), b.copy()
    a0[11], b0[11] = np.float32(-0.0), np.float32(0.0)
    z = ose.evaluate(ose.gather_rows({1: {"bed": a0[None]}, 2: {"bed": b0[None]}}, ["bed"]), gt)
    assert z["prec"]["bed"].tolist() == [1.0, 0.5]


def test_class_without_detection_has_ap_zero():
    from oracle import sunrgbd_eval as ose
    g, a, _ = _tie_case()
    r = ose.evaluate({"bed": ose.gather_rows({1: {"bed": a[None]}}, ["bed"])["bed"]}, {"bed": {1: [g]}, "sofa": {1: [g]}})
    assert r["ap"]["sofa"] == 0.0 and len(r["rec"]["sofa"]) == 0 and r["npos"]["sofa"] == 1
    assert r["ap"]["bed"] == 1.0 and r["lines"] == ["bed: 1.00000", "sofa: 0.00000", "mean_AP: 0.50000"]


def _args(seg=(0, 1, 3), gcls=(0, 3), dcls=(0, 2)):
    from frustum_convnet_b200 import _lib
    keep = [np.asarray(seg, np.int32), np.asarray(gcls, np.int32), np.asarray(dcls, np.int32), np.zeros(64)]
    a = _lib.SunrgbdEvalArgs()
    a.num_classes, a.num_gt, a.num_gt_segments, a.num_det = len(gcls) - 1, int(gcls[-1]), len(seg) - 1, int(dcls[-1])
    a.ovthresh = 0.25
    dummy = keep[3].ctypes.data
    for f in ("gt_corners", "det_corners", "det_scores", "det_segments", "gt_segment_offsets", "gt_class_offsets",
              "det_class_offsets", "workspace", "rec", "prec", "result"):
        setattr(a, f, dummy)
    a.host_gt_segment_offsets, a.host_gt_class_offsets, a.host_det_class_offsets = (k.ctypes.data for k in keep[:3])
    a.workspace_bytes = 1 << 40
    return a, keep


def test_argument_validation_without_gpu():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    entries = (lib.fcn_sunrgbd_eval_match, lib.fcn_sunrgbd_eval_curves)
    for fn in entries:
        assert fn(None, None) == -1
        assert b"NULL args" in lib.fcn_last_error()
    assert lib.fcn_sunrgbd_eval_workspace_bytes(None) == -1

    def expect(mutate, msg):
        a, keep = _args()
        mutate(a, keep)
        assert lib.fcn_sunrgbd_eval_workspace_bytes(ctypes.byref(a)) == -1
        assert msg in lib.fcn_last_error(), lib.fcn_last_error()
        for fn in entries:
            assert fn(ctypes.byref(a), None) == -1
            assert msg in lib.fcn_last_error(), lib.fcn_last_error()

    expect(lambda a, k: setattr(a, "num_det", -1), b"negative count")
    expect(lambda a, k: setattr(a, "num_classes", 5000), b"too many records")
    expect(lambda a, k: setattr(a, "gt_corners", None), b"NULL pointer")
    expect(lambda a, k: setattr(a, "det_segments", None), b"NULL pointer")
    expect(lambda a, k: setattr(a, "host_gt_class_offsets", None), b"NULL host offsets")

    def decreasing(a, k):
        k[0][:] = (0, 2, 1)
    expect(decreasing, b"never decrease")

    def wrong_total(a, k):
        k[2][1] = 3
    expect(wrong_total, b"end at num_gt / num_det")

    def crossing(a, k):                                  # class boundary at 2, segments at 0, 1, 3
        a.num_classes = 2
        k[1].resize(3, refcheck=False)
        k[1][:] = (0, 2, 3)
        k[2].resize(3, refcheck=False)
        k[2][:] = (0, 1, 2)
        a.host_gt_class_offsets, a.host_det_class_offsets = k[1].ctypes.data, k[2].ctypes.data
    expect(crossing, b"crosses a class boundary")

    for field in ("workspace", "result", "rec"):          # not needed by the size query, required by the entries
        a, keep = _args()
        setattr(a, field, None)
        for fn in entries:
            assert fn(ctypes.byref(a), None) == -1
            assert b"NULL workspace or output" in lib.fcn_last_error()


def test_cpu_device_raises():
    from frustum_convnet_b200.sunrgbd_eval import SunrgbdGroundTruth
    with pytest.raises(RuntimeError):
        SunrgbdGroundTruth({"bed": (np.zeros((0, 8, 3)), np.zeros(0))}, device="cpu")
