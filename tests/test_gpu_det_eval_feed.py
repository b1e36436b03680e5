"""GPU: ``evaluate_collected`` (the evaluators fed from DetectionCollector.finalize_device() by
csrc/det_eval_feed.cu) against ``evaluate(collector.finalize())``.

KITTI: every record field but alpha bit-identical to detection_records; alpha within one '%.4f' step, identical
where numpy's float32 atan2 is correctly rounded; the 41-point image / ground / 3-D precision vectors and the printed
AP bit-identical (they do not read alpha); AOS within 1e-6.  SUN-RGBD: corners within 2 float32 ulps of the corner
magnitude; rec / prec / AP bit-identical on sets whose overlaps keep a margin from ovthresh and have no near tie
(oracle/sunrgbd_synth.margins_ok); on unconstrained sets AP within 1e-4, with the differing TP flags reported."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR
from det_feed_sets import collector_for, kitti_set

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ helpers
def kitti_feed_records(ev, col_dev):
    """The records fcn_det_kitti_records writes, read back, with the plan's offsets."""
    from frustum_convnet_b200 import _lib
    from frustum_convnet_b200._host import upload
    seg_dst, seg_code, det_off = ev.gather_plan(col_dev)
    n = int(det_off[-1])
    buf, (p_dst, p_code, _) = upload([seg_dst, seg_code, det_off], ev.device)
    out = torch.empty((max(n, 1), 14), dtype=torch.float64, device=ev.device)
    a = col_dev.feed_args(seg_dst, seg_code, n, (p_dst, p_code))
    a.records = out.data_ptr()
    _lib.call("fcn_det_kitti_records", C.byref(a), torch.cuda.current_stream().cuda_stream)
    return out[:n].cpu().numpy(), det_off


def host_kitti_records(ev, dets):
    from frustum_convnet_b200.kitti_eval import detection_records
    """-> (the records of the dict path, in its order, and the float32 rows they came from)."""
    per_image = [[] for _ in ev.gt.image_ids]
    for idx, by_class in dets.items():
        for ct, d in by_class.items():
            if len(d):
                per_image[ev.gt.index[int(idx)]].append((detection_records(d, ct), d))
    if not any(per_image):
        return np.zeros((0, 14)), np.zeros((0, 12), np.float32)
    return (np.concatenate([r for p in per_image for r, _ in p]), np.concatenate([d for p in per_image for _, d in p]))


def check_kitti(ev, col):
    cd = col.finalize_device()
    dets = cd.to_dict()
    got, _ = kitti_feed_records(ev, cd)
    want, rows = host_kitti_records(ev, dets)
    assert got.shape == want.shape
    cols = [0] + list(range(2, 14))
    assert np.array_equal(got[:, cols].view(np.int64), want[:, cols].view(np.int64))
    assert (np.abs(got[:, 1] - want[:, 1]) <= 1e-4 + 1e-9).all()
    # alpha identical wherever numpy's float32 atan2 is the correctly rounded value
    x, z = rows[:, 4], rows[:, 6]
    same = np.arctan2(z, x) == np.arctan2(z.astype(np.float64), x.astype(np.float64)).astype(np.float32)
    assert np.array_equal(got[same, 1].view(np.int64), want[same, 1].view(np.int64))
    res_d = ev.evaluate_collected(cd)
    res_h = ev.evaluate(dets)
    compare_kitti_results(res_d, res_h)
    return got, want, res_d


def compare_kitti_results(a, b):
    assert a.evaluated == b.evaluated and a.compute_aos == b.compute_aos
    for m in a.precision:
        assert a.precision[m].keys() == b.precision[m].keys()
        for c in a.precision[m]:
            assert np.array_equal(a.precision[m][c].view(np.int64), b.precision[m][c].view(np.int64)), (m, c)
            assert np.array_equal(a.ap[m][c], b.ap[m][c]), (m, c)
            assert np.array_equal(a.n_thresholds[m][c], b.n_thresholds[m][c])
            assert np.array_equal(a.n_gt[m][c], b.n_gt[m][c])
    assert a.aos.keys() == b.aos.keys()
    for c in a.aos:
        assert np.abs(a.aos[c] - b.aos[c]).max() <= 1e-6
    lines_a = [l for l in a.lines() if "orientation" not in l]
    assert lines_a == [l for l in b.lines() if "orientation" not in l]


def kitti_gt(image_ids, records):
    from frustum_convnet_b200.kitti_eval import KittiEvaluator, KittiGroundTruth
    return KittiEvaluator(KittiGroundTruth(image_ids, records))


def sun_gt(gt_rows, gt_ids, classes, image_ids=None):
    from frustum_convnet_b200.sunrgbd_eval import SunrgbdEvaluator, SunrgbdGroundTruth, gt_corners
    return SunrgbdEvaluator(SunrgbdGroundTruth({c: (gt_corners(gt_rows[c]), gt_ids[c]) for c in classes}, image_ids))


def tp_flags(res, c):
    r = res.rec[c]
    return np.diff(np.concatenate([[0.0], r])) > 0 if len(r) else np.zeros(0, bool)


def check_sunrgbd(ev, col, exact, ovthresh=0.25):
    from frustum_convnet_b200.sunrgbd_eval import det_corners
    cd = col.finalize_device()
    dets = cd.to_dict()
    res_d = ev.evaluate_collected(cd, ovthresh=ovthresh)
    res_h = ev.evaluate(dets, ovthresh=ovthresh)
    # the corners: the device's, read through the plan, against det_corners
    seg_dst, seg_gt, det_off = ev.gather_plan(cd)
    rows = cd.rows[:cd.num_rows].cpu().numpy()
    for s in range(cd.num_segments):
        d, k0, kc = seg_dst[s], cd.host_seg_offsets[s], cd.host_keep_count[s]
        if d < 0 or kc == 0:
            continue
        want = det_corners(rows[k0:k0 + kc])
        got = device_corners(cd, s)
        tol = 2 * np.spacing(np.float32(np.abs(want).max(axis=(1, 2)))).astype(np.float64)
        assert (np.abs(got - want).max(axis=(1, 2)) <= tol).all()
    assert res_d.classes == res_h.classes
    flips = 0
    for c in res_h.classes:
        assert res_d.nd[c] == res_h.nd[c] and res_d.npos[c] == res_h.npos[c]
        if exact:
            assert np.array_equal(res_d.rec[c].view(np.int64), res_h.rec[c].view(np.int64)), c
            assert np.array_equal(res_d.prec[c].view(np.int64), res_h.prec[c].view(np.int64)), c
            assert res_d.ap[c] == res_h.ap[c], c
        else:
            assert abs(res_d.ap[c] - res_h.ap[c]) <= 1e-4, c
            flips += int((tp_flags(res_d, c) != tp_flags(res_h, c)).sum())
    if not exact:
        print("SUN-RGBD: %d TP flags differ between the device and host corners" % flips)
    return res_d, res_h


_CORNER_CACHE = {}


def device_corners(cd, s):
    """Corners of segment s as fcn_det_sunrgbd_feed writes them (every segment written, in segment order)."""
    key = id(cd)
    if key not in _CORNER_CACHE:
        from frustum_convnet_b200 import _lib
        from frustum_convnet_b200._host import upload
        S = cd.num_segments
        kc = cd.host_keep_count.astype(np.int64)
        seg_dst = (np.cumsum(kc) - kc).astype(np.int32)
        seg_val = np.full(S, -1, np.int32)
        n = int(kc.sum())
        buf, (p_dst, p_val) = upload([seg_dst, seg_val], cd.device)
        out = torch.empty(max(n, 1) * 26, dtype=torch.float64, device=cd.device)
        a = cd.feed_args(seg_dst, seg_val, n, (p_dst, p_val))
        a.corners, a.scores, a.segments = out.data_ptr(), out.data_ptr() + 192 * n, out.data_ptr() + 200 * n
        _lib.call("fcn_det_sunrgbd_feed", C.byref(a), torch.cuda.current_stream().cuda_stream)
        _CORNER_CACHE.clear()
        _CORNER_CACHE[key] = (cd, seg_dst, out[:24 * n].cpu().numpy().reshape(n, 8, 3))
    _, seg_dst, cor = _CORNER_CACHE[key]
    return cor[seg_dst[s]: seg_dst[s] + cd.host_keep_count[s]]


# ------------------------------------------------------------------------------------------------ fixtures
def _golden_collector(name, dataset, run):
    from oracle.make_golden_detect import batches
    from test_detect_cpu import fixture_runs
    from frustum_convnet_b200.detect import DetectionCollector
    g = dict(np.load(os.path.join(GOLDEN_DIR, "detect_%s.npz" % name)))
    ids, types = [int(i) for i in g["id_list"]], [str(t) for t in g["type_list"]]
    method, use_ref, use_rgb, want = fixture_runs(g)[run]
    col = DetectionCollector(ids, types, g["box2d"], dataset=dataset, method=method, thresh=float(g["thresh"]))
    for first, outs, rot, rgb, ref in batches(g, use_ref, use_rgb):
        d = {"rot_angle": torch.from_numpy(np.asarray(rot).reshape(-1, 1).copy()).cuda()}
        if rgb is not None:
            d["rgb_prob"] = torch.from_numpy(np.asarray(rgb).reshape(-1, 1).copy()).cuda()
        if ref is not None:
            d["ref_center"] = torch.from_numpy(np.asarray(ref).copy()).cuda()
        col.add(tuple(torch.from_numpy(np.ascontiguousarray(o)).cuda() for o in outs), d, first=first)
    return col, sorted(set(ids)), len(fixture_runs(g))


@pytest.mark.parametrize("run", range(4))
def test_kitti_golden_detections(run):
    from oracle import kitti_synth as ks
    col, det_ids, _ = _golden_collector("kitti", "KITTI", run)
    g = np.load(os.path.join(GOLDEN_DIR, "kitti_eval.npz"))
    labels = [ks.parse_label_lines(str(t).splitlines()) for t in g["main_labels"]]
    ids = det_ids + [1000 + k for k in range(len(labels) - len(det_ids))]
    check_kitti(kitti_gt(ids, labels), col)


@pytest.mark.parametrize("run", range(4))
def test_sunrgbd_golden_detections(run):
    col, det_ids, _ = _golden_collector("sunrgbd", "SUNRGBD", run)
    g = np.load(os.path.join(GOLDEN_DIR, "sunrgbd_eval.npz"))
    classes = [str(c) for c in g["real_classes"]]
    counts = np.concatenate([[0], np.cumsum(g["real_gt_class_counts"])])
    uniq = sorted(set(g["real_gt_ids"].tolist()))
    remap = {u: (det_ids[k] if k < len(det_ids) else 10000 + k) for k, u in enumerate(uniq)}
    rows = {c: g["real_gt_rows"][counts[i]:counts[i + 1]] for i, c in enumerate(classes)}
    ids = {c: np.array([remap[int(v)] for v in g["real_gt_ids"][counts[i]:counts[i + 1]]]) for i, c in
           enumerate(classes)}
    check_sunrgbd(sun_gt(rows, ids, classes), col, exact=False)


# ------------------------------------------------------------------------------------------------ synthetic KITTI
def test_kitti_thousands_of_images():
    gts, dets = kitti_set(2000, seed=3)
    _, want, _ = check_kitti(kitti_gt(list(range(len(gts))), gts), collector_for(dets, "KITTI"))
    assert len(want) > 10000


def test_kitti_one_row_zero_rows_and_an_undetected_class():
    gts, dets = kitti_set(40, seed=4)
    ev = kitti_gt(list(range(len(gts))), gts)
    one = {7: {"Car": next(d["Car"][:1] for d in dets.values() if "Car" in d)}}
    check_kitti(ev, collector_for(one, "KITTI"))
    # zero kept rows: every list is empty (rows dropped by the decode's size rule)
    check_kitti(ev, collector_for({3: {"Car": np.zeros((0, 12))}, 5: {"Pedestrian": np.zeros((0, 12))}}, "KITTI"))
    # no cyclist detected at all, plus a frustum of an image outside the ground truth that is never added
    nocyc = {i: {c: d for c, d in by.items() if c != "Cyclist"} for i, by in dets.items()}
    got, _, res = check_kitti(ev, collector_for(nocyc, "KITTI", extra_frustums=[(999, "Car")]))
    assert "cyclist" not in res.ap["3d"]


def test_kitti_image_outside_the_ground_truth_raises():
    gts, dets = kitti_set(10, seed=5)
    ev = kitti_gt(list(range(len(gts))), gts)
    bad = dict(dets)
    bad[12345] = {"Car": np.asarray(next(iter(dets.values())).get("Car", np.zeros((0, 12))))}
    cd = collector_for(bad, "KITTI").finalize_device()
    with pytest.raises(KeyError):
        ev.evaluate_collected(cd)
    with pytest.raises(KeyError):
        ev.evaluate(cd.to_dict())


def test_kitti_quantization_ties():
    """Rows whose fields sit on '%.4f' / '%f' ties: odd multiples of 1/32 (x * 1e4 = k + 1/2) and of 1/128 for the
    score (x * 1e6 = k + 1/2); ty = (ty - h/2) + h/2 is exact for them."""
    rng = np.random.default_rng(6)
    n = 64
    odd = lambda lo, hi, den: (2 * rng.integers(lo, hi, n) + 1) / den
    rows = np.zeros((n, 12), np.float32)
    rows[:, 0], rows[:, 1] = odd(100, 200, 32), odd(50, 100, 32)
    rows[:, 2], rows[:, 3] = rows[:, 0] + rng.integers(5, 20, n) / 16, rows[:, 1] + rng.integers(5, 20, n) / 16
    rows[:, 4], rows[:, 5], rows[:, 6] = odd(-300, 300, 32), odd(0, 40, 32), odd(100, 1000, 32)
    rows[:, 7], rows[:, 8], rows[:, 9] = odd(20, 30, 32), odd(20, 30, 32), odd(50, 70, 32)
    rows[:, 10], rows[:, 11] = odd(-40, 40, 32), odd(0, 63, 128)
    assert ((rows[:, :11].astype(np.float64) * 1e4) % 1 == 0.5).all()
    assert ((rows[:, 11].astype(np.float64) * 1e6) % 1 == 0.5).all()
    gts, _ = kitti_set(3, seed=6)
    ev = kitti_gt([0, 1, 2], gts)
    got, want, _ = check_kitti(ev, collector_for({0: {"Car": rows[:32]}, 2: {"Pedestrian": rows[32:]}}, "KITTI"))
    assert len(got) == n


@pytest.mark.parametrize("method", ["top", "nms"])
def test_kitti_methods(method):
    gts, dets = kitti_set(300, seed=7)
    check_kitti(kitti_gt(list(range(len(gts))), gts), collector_for(dets, "KITTI", method=method))


def test_graph_captured_add_and_two_streams():
    gts, dets = kitti_set(30, seed=8)
    ev = kitti_gt(list(range(len(gts))), gts)
    ref = collector_for(dets, "KITTI")
    want = ref.finalize()
    # the same rows appended by a captured add, replayed once
    col = collector_for(dets, "KITTI")
    col.reset()
    side = torch.cuda.Stream()
    F = col.num_frustums
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        outs, d = _outputs_of(dets)
        col.add(outs, d, first=0)          # warm-up outside the graph
    torch.cuda.current_stream().wait_stream(side)
    col.reset()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        col.add(outs, d, first=0)
    graph.replay()
    cd = col.finalize_device()
    assert _same(cd.to_dict(), want)
    compare_kitti_results(ev.evaluate_collected(cd), ev.evaluate(want))
    # rows added on two streams, evaluated on a third
    col = collector_for(dets, "KITTI")
    col.reset()
    s1, s2, s3 = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    half = F // 2
    for s, lo, hi in ((s1, 0, half), (s2, half, F)):
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            o, dd = _outputs_of(dets, lo, hi)
            col.add(o, dd, first=lo)
    cd = col.finalize_device()
    assert _same(cd.to_dict(), want)
    with torch.cuda.stream(s3):
        res = ev.evaluate_collected(cd, stream=s3)
    compare_kitti_results(res, ev.evaluate(want))


def _outputs_of(dets, lo=0, hi=None):
    """The model outputs collector_for feeds, for frustums [lo, hi)."""
    rows = np.concatenate([np.asarray(d, np.float32).reshape(-1, 12) for by in dets.values() for d in by.values()])
    hi = len(rows) if hi is None else hi
    r = rows[lo:hi]
    F = len(r)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()
    cls = np.zeros((F, 1, 2), np.float32)
    cls[:, 0, 1] = r[:, 11]
    center = np.stack([r[:, 4], r[:, 5] - r[:, 7] * np.float32(0.5), r[:, 6]], 1).reshape(F, 1, 3)
    sp = np.zeros((F, 1, 1), np.float32)
    return ((t(cls), t(center), t(r[:, 10].reshape(F, 1)), t(r[:, [9, 8, 7]].reshape(F, 1, 3)), t(sp), t(sp)),
            {"rot_angle": t(np.zeros((F, 1))), "rgb_prob": t(np.zeros((F, 1)))})


def _same(a, b):
    if list(a) != list(b):
        return False
    for i in a:
        if list(a[i]) != list(b[i]):
            return False
        for c in a[i]:
            if not np.array_equal(a[i][c].view(np.int32), b[i][c].view(np.int32)):
                return False
    return True


def test_finalize_after_finalize_device():
    col, _, _ = _golden_collector("kitti", "KITTI", 0)
    first = col.finalize()
    cd = col.finalize_device()
    again = col.finalize()
    assert _same(first, again) and _same(cd.to_dict(), first)
    from test_detect_cpu import fixture_runs
    g = dict(np.load(os.path.join(GOLDEN_DIR, "detect_kitti.npz")))
    want = fixture_runs(g)[0][3]
    assert list((i, c) for i in first for c in first[i]) == list(want)


# ------------------------------------------------------------------------------------------------ synthetic SUN-RGBD
def _sun_set(n_images, seed, check_margins, **kw):
    from oracle import sunrgbd_synth as ss
    from frustum_convnet_b200.sunrgbd_eval import CLASS_NAMES
    classes = list(CLASS_NAMES)
    gt_rows, gt_ids, dets = ss.make_set(seed, n_images, classes, check_margins=check_margins, **kw)
    return classes, gt_rows, gt_ids, dets


def test_sunrgbd_margin_sets_are_bit_identical():
    classes, gt_rows, gt_ids, dets = _sun_set(300, 11, True)
    ev = sun_gt(gt_rows, gt_ids, classes)
    res_d, _ = check_sunrgbd(ev, collector_for(dets, "SUNRGBD"), exact=True)
    assert sum(res_d.nd.values()) > 500 and res_d.mean_ap > 0


def test_sunrgbd_unconstrained_set():
    classes, gt_rows, gt_ids, dets = _sun_set(500, 12, False, gt_mean=0.26, fp_rate=2.5)
    check_sunrgbd(sun_gt(gt_rows, gt_ids, classes), collector_for(dets, "SUNRGBD"), exact=False)


def test_sunrgbd_gather_order_is_per_class_dict_order():
    """Frustums (A, chair), (B, table), (A, table): the table rows gather A before B."""
    classes, gt_rows, gt_ids, dets = _sun_set(2, 13, True)
    A, B = 1, 2
    base = np.concatenate([d for by in dets.values() for d in by.values()])
    ev = sun_gt(gt_rows, gt_ids, classes)
    # frustum order (A, chair), (B, table), (A, table)
    col = _ordered_collector([(A, "chair", base[:2]), (B, "table", base[2:4]), (A, "table", base[4:7])])
    cd = col.finalize_device()
    seg_dst, _, det_off = ev.gather_plan(cd)
    t = ev.gt.class_index["table"]
    segs = [s for s in range(cd.num_segments) if cd.segments[s][1] == "table"]
    a_seg = next(s for s in segs if cd.segments[s][0] == A)
    b_seg = next(s for s in segs if cd.segments[s][0] == B)
    assert seg_dst[a_seg] == det_off[t] and seg_dst[b_seg] == det_off[t] + 3
    check_sunrgbd(ev, col, exact=True)


def _ordered_collector(items):
    """SUN-RGBD frustums of the (image, class, rows) items in the given order, one frustum per row."""
    from frustum_convnet_b200.detect import DetectionCollector
    ids, types, rr = [], [], []
    for idx, c, rows in items:
        for r in rows:
            ids.append(idx)
            types.append(c)
            rr.append(r)
    rr = np.asarray(rr, np.float32)
    F = len(rr)
    col = DetectionCollector(ids, types, rr[:, :4].astype(np.float64), dataset="SUNRGBD", method="top")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()
    cls = np.zeros((F, 1, 2))
    cls[:, 0, 1] = 1
    outs = (t(cls), t(rr[:, 4:7].reshape(F, 1, 3)), t(rr[:, 10].reshape(F, 1)),
            t(rr[:, 7:10].reshape(F, 1, 3)), t(rr[:, 11].reshape(F, 1, 1)), t(rr[:, 11].reshape(F, 1, 1)))
    col.add(outs, {"rot_angle": t(np.zeros((F, 1))), "rgb_prob": t(np.zeros((F, 1)))}, first=0)
    return col


def test_sunrgbd_edges():
    classes, gt_rows, gt_ids, dets = _sun_set(60, 14, True)
    ev = sun_gt(gt_rows, gt_ids, classes, image_ids=list(range(1, 61)))
    first = next(iter(dets))
    c0 = next(iter(dets[first]))
    check_sunrgbd(ev, collector_for({first: {c0: dets[first][c0][:1]}}, "SUNRGBD"), exact=True)      # one row
    check_sunrgbd(ev, collector_for({first: {c0: np.zeros((0, 12))}}, "SUNRGBD"), exact=True)        # zero rows
    # a class never detected and one without ground truth ("lamp"), plus a never-added frustum
    nochair = {i: {c: d for c, d in by.items() if c != "chair"} for i, by in dets.items()}
    nochair[first]["lamp"] = dets[first][c0][:2]
    res_d, _ = check_sunrgbd(ev, collector_for(nochair, "SUNRGBD", extra_frustums=[(777, "chair")]), exact=True)
    assert res_d.nd["chair"] == 0
    # an image in neither the ground truth nor image_ids raises
    bad = {**dets, 5000: {c0: dets[first][c0][:1]}}
    with pytest.raises(KeyError):
        ev.evaluate_collected(collector_for(bad, "SUNRGBD").finalize_device())


def test_sunrgbd_non_finite_rows_raise():
    classes, gt_rows, gt_ids, dets = _sun_set(4, 15, True)
    first = next(iter(dets))
    c0 = next(iter(dets[first]))
    rows = np.array(dets[first][c0][:2])
    rows[1, 4] = np.inf
    ev = sun_gt(gt_rows, gt_ids, classes)
    cd = collector_for({first: {c0: rows}}, "SUNRGBD").finalize_device()
    with pytest.raises(ValueError):
        ev.evaluate_collected(cd)
    with pytest.raises(ValueError):
        ev.evaluate(cd.to_dict())
