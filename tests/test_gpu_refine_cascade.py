"""GPU: the refinement stage fed from the first stage's device detections (csrc/refine_jobs.cu via
RefineFrustumExtractor.from_collected / from_matched_collected) against the dict path on the same collector
(from_detections / from_matched_detections of finalize()'s dict): job order, kept set, points, labels and quantized
values exactly, the angle-derived values within 4 ulp, TrainBatchBuilder.from_frustums batches from the device records
against the host table, and a refinement forward of each into a second collector."""
import numpy as np
import pytest
import torch

from det_feed_sets import collector_for

pytestmark = pytest.mark.gpu

ANGLE_ULP = 4


def _dets(results, ids):
    """Result lines {idx: [line]} -> the collector rows {idx: {class: (n, 12) float32}} of the images in ids."""
    from oracle import kitti_refine_synth as krs
    dets = {}
    for i, objs in krs.objects(results).items():
        if i not in ids:
            continue
        rows = {}
        for o in objs:
            rows.setdefault(o.type, []).append(list(o.box2d) + list(o.t) + [o.h, o.w, o.l, o.ry, o.score])
        dets[i] = {c: np.array(r, np.float32) for c, r in rows.items()}
    return dets


def _scene(seed, n_frames=4, n_points=30000, extra_images=()):
    from oracle import kitti_refine_synth as krs
    scans, calibs, hws, labels, results = krs.large_scene(seed, n_frames=n_frames, n_points=n_points)
    ids = sorted(scans)
    col = collector_for(_dets(results, ids), "KITTI", extra_frustums=[(i, "Car") for i in extra_images])
    return scans, calibs, hws, ids, krs.objects(labels), col


def _ulp(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b)))


def _same(a, b, what):
    """a: the dict path's RefineFrustums, b: the collected path's.  Returns the bit-identical share of the angle-derived
    values."""
    assert len(a) == len(b), what
    assert torch.equal(a.offsets, b.offsets) and torch.equal(a.points, b.points), what
    assert np.array_equal(a.counts, b.counts), what
    assert (a.label is None) == (b.label is None) and (a.label is None or torch.equal(a.label, b.label)), what
    assert a.id_list == b.id_list and a.type_list == b.type_list, what
    assert np.array(a.box2d_list).tobytes() == np.array(b.box2d_list).tobytes(), what
    assert a.prob_list == b.prob_list, what
    for n in ("pred_box3d_size_list", "pred_box3d_angle_list"):
        assert np.array(getattr(a, n)).tobytes() == np.array(getattr(b, n)).tobytes(), (what, n)
    if a.has_labels:
        for n in ("box3d_list", "heading_list", "size_list"):
            assert np.array(getattr(a, n)).tobytes() == np.array(getattr(b, n)).tobytes(), (what, n)
    same = total = 0
    for n in ("frustum_angle_list", "pred_box3d_list"):
        x, y = np.array(getattr(a, n)).reshape(-1), np.array(getattr(b, n)).reshape(-1)
        assert (_ulp(x, y) <= ANGLE_ULP).all(), (what, n, float(_ulp(x, y).max()))
        same += int((x == y).sum())
        total += x.size
    return same, total


def _both(x, mode, scans, calibs, hws, ids, col, gt=None, stream=None):
    collected = col.finalize_device()
    if mode == "det":
        a = x.from_detections(scans, calibs, hws, ids, collected.to_dict())
        b = x.from_collected(scans, calibs, hws, ids, collected, stream=stream)
    else:
        a = x.from_matched_detections(scans, calibs, hws, ids, collected.to_dict(), gt, remove_diff=True)
        b = x.from_matched_collected(scans, calibs, hws, ids, collected, gt, remove_diff=True, stream=stream)
    return a, b


@pytest.mark.parametrize("mode,whitelist", [("det", ("Car",)), ("det", ("Car", "Pedestrian", "Cyclist")),
                                            ("matched", ("Car",)), ("matched", ("Pedestrian", "Cyclist"))])
def test_collected_matches_the_dict_path(mode, whitelist):
    from frustum_convnet_b200 import refine_extract as rx
    scans, calibs, hws, ids, gt, col = _scene(31, n_frames=6)
    a, b = _both(rx.RefineFrustumExtractor(whitelist), mode, scans, calibs, hws, ids, col, gt)
    assert len(a) > 0
    same, total = _same(a, b, mode)
    print("%s %s: %d frustums, angle-derived values bit-identical %d / %d" % (mode, whitelist, len(a), same, total))
    assert torch.equal(b.frustum_angle.cpu(), torch.from_numpy(np.array(b.frustum_angle_list)))


@pytest.mark.parametrize("mode", ["det", "matched"])
def test_segment_tables_of_one_and_3769_images(mode):
    from frustum_convnet_b200 import refine_extract as rx
    scans, calibs, hws, ids, gt, col = _scene(32, n_frames=1)
    x = rx.RefineFrustumExtractor(("Car", "Pedestrian"))
    a, b = _both(x, mode, scans, calibs, hws, ids, col, gt)
    assert len(a) > 0
    _same(a, b, "one image")
    # a validation-sized table: 3769 images, most without detections (their frustums never added), some listed twice
    others = [i for i in range(3769) if i not in ids]
    scans, calibs, hws, ids, gt, col = _scene(33, n_frames=5, extra_images=others)
    image_ids = list(range(3769)) + ids[:1]
    gt = {i: gt.get(i, []) for i in image_ids}
    a, b = _both(x, mode, scans, calibs, hws, image_ids, col, gt)
    assert len(a) > 0
    _same(a, b, "3769 images")


def test_zero_kept_rows():
    from frustum_convnet_b200 import refine_extract as rx
    scans, calibs, hws, ids, gt, col = _scene(34, n_frames=2)
    for whitelist in (("Cyclist", "Van"), ("Truck",)):
        x = rx.RefineFrustumExtractor(whitelist)
        for mode in ("det", "matched"):
            a, b = _both(x, mode, scans, calibs, hws, ids, col, gt)
            _same(a, b, (whitelist, mode))
            if whitelist == ("Truck",):
                assert len(b) == 0 and b.points.shape == (0, 4) and b.offsets.tolist() == [0] and b.id_list == []
    # detections of images outside image_ids are ignored, as the dict path ignores them
    a, b = _both(rx.RefineFrustumExtractor(("Car",)), "det", scans, calibs, hws, [1, 2], col)
    assert len(a) == len(b) == 0
    # a collector whose rows the decode drops (sizes below 0.01): no kept row at all
    empty = collector_for({ids[0]: {"Car": np.zeros((2, 12), np.float32)}}, "KITTI")
    collected = empty.finalize_device()
    assert collected.host_keep_count.sum() == 0
    fr = rx.RefineFrustumExtractor(("Car",)).from_collected(scans, calibs, hws, ids, collected)
    assert len(fr) == 0 and fr.prob_list == [] and fr.pred_box3d_list == []


def test_two_streams():
    from frustum_convnet_b200 import refine_extract as rx
    scans, calibs, hws, ids, gt, col = _scene(35, n_frames=4)
    x = rx.RefineFrustumExtractor(("Car", "Pedestrian"))
    collected = col.finalize_device()
    base = x.from_collected(scans, calibs, hws, ids, collected)
    want = [p.tobytes() for p in base.input_list()]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    dev_scans = {k: torch.from_numpy(v).cuda() for k, v in scans.items()}
    torch.cuda.synchronize()
    f1 = x.from_collected(dev_scans, calibs, hws, ids, collected, stream=s1)
    f2 = x.from_matched_collected(dev_scans, calibs, hws, ids, collected, gt, stream=s2)
    assert f1.stream is s1 and f2.stream is s2
    assert [p.tobytes() for p in f1.input_list()] == want
    assert np.array(f1.pred_box3d_list).tobytes() == np.array(base.pred_box3d_list).tobytes()
    ref = x.from_matched_detections(scans, calibs, hws, ids, collected.to_dict(), gt)
    _same(ref, f2, "matched on a side stream")


def _bad_collector(ids, row):
    good = np.array([[100, 120, 180, 170, 2.0, 1.6, 20.0, 1.5, 1.6, 3.9, 0.3, 0.9]], np.float32)
    return collector_for({ids[0]: {"Car": np.concatenate([good, row[None]]), "Pedestrian": good},
                          ids[1]: {"Car": good}}, "KITTI")


@pytest.mark.parametrize("what", ["nan_x", "nan_ry", "zero_l", "negative_h"])
def test_bad_rows_raise_what_the_dict_path_raises(what):
    from frustum_convnet_b200 import refine_extract as rx
    scans, calibs, hws, ids, gt, _ = _scene(36, n_frames=2, n_points=20000)
    row = np.array([100, 120, 180, 170, 2.0, 1.6, 20.0, 1.5, 1.6, 3.9, 0.3, 0.9], np.float32)
    col = _bad_collector(ids, row)
    collected = col.finalize_device()           # the second Car row of the first image is rewritten in place
    r = collected.rows[:collected.num_rows]
    k = int(collected.host_seg_offsets[0]) + 1
    field = {"nan_x": 4, "nan_ry": 10, "zero_l": 9, "negative_h": 7}[what]
    r[k, field] = {"nan_x": float("nan"), "nan_ry": float("nan"), "zero_l": 0.0, "negative_h": -1.0}[what]
    x = rx.RefineFrustumExtractor(("Car",))
    with pytest.raises(ValueError) as e1:
        x.from_detections(scans, calibs, hws, ids, collected.to_dict())
    with pytest.raises(ValueError) as e2:
        x.from_collected(scans, calibs, hws, ids, collected)
    assert str(e1.value) == str(e2.value) and "row 1" in str(e2.value)
    m = x.from_matched_detections if what.startswith("nan") else None
    if m is not None:                            # a non-finite box raises in matched mode too, matched or not
        with pytest.raises(ValueError) as e1:
            m(scans, calibs, hws, ids, collected.to_dict(), gt)
        with pytest.raises(ValueError) as e2:
            x.from_matched_collected(scans, calibs, hws, ids, collected, gt)
        assert str(e1.value) == str(e2.value)
    else:                                        # an unmatched flat box is no error in matched mode
        a = x.from_matched_detections(scans, calibs, hws, ids, collected.to_dict(), gt)
        b = x.from_matched_collected(scans, calibs, hws, ids, collected, gt)
        _same(a, b, what)


@pytest.mark.parametrize("mode", ["det", "matched"])
def test_batches_and_refinement_forward_from_both_tables(mode):
    from train_ref import make_model
    from frustum_convnet_b200 import config
    from frustum_convnet_b200 import refine_extract as rx
    from frustum_convnet_b200.detect import DetectionCollector
    from frustum_convnet_b200.train_inputs import TrainBatchBuilder
    scans, calibs, hws, ids, gt, col = _scene(37, n_frames=6)
    a, b = _both(rx.RefineFrustumExtractor(("Car", "Pedestrian", "Cyclist")), mode, scans, calibs, hws, ids, col, gt)
    assert len(a) > 0 and b.frustum_records is not None
    cfg, _ = config.load_workload("refine_car")
    strides, N = list(cfg.DATA.STRIDE), int(cfg.DATA.NUM_SAMPLES)
    ta = TrainBatchBuilder.from_frustums(a, "refine", strides=strides, npoints=N)
    tb = TrainBatchBuilder.from_frustums(b, "refine", strides=strides, npoints=N)
    assert tb.d_frustums is b.frustum_records              # installed as the extractor wrote them
    assert np.array_equal(ta.T_of, tb.T_of)
    idx = np.arange(len(a))
    draws = ta.draw(idx, np.random.RandomState(3))
    ba = {k: v.clone() for k, v in ta.build(idx, draws).items()}
    bb = tb.build(idx, draws)
    assert sorted(ba) == sorted(bb)
    same = total = 0
    for k in ba:
        x, y = ba[k].cpu().numpy(), bb[k].cpu().numpy()
        assert x.shape == y.shape and x.dtype == y.dtype, k
        if x.dtype.kind == "f":
            d = np.abs(x.astype(np.float64) - y) / np.spacing(np.maximum(np.abs(x), np.abs(y)).astype(np.float32))
            assert (d <= 1).all(), (k, float(d.max()))
            same += int((x.view(np.int32) == y.view(np.int32)).sum())
            total += x.size
        else:
            assert np.array_equal(x, y), k
    assert same >= 0.999 * total, (same, total)
    print("%s: batch float values bit-identical %d / %d" % (mode, same, total))
    m2 = make_model("refine_car", 5).eval()
    outs = []
    labels = ("cls_label", "box3d_center", "box3d_heading", "box3d_size", "size_class")
    for fr, data in ((a, ba), (b, bb)):
        data = {k: v for k, v in data.items() if k not in labels}       # inference: the model returns the heads
        with torch.no_grad():
            out = m2(data)
        c2 = DetectionCollector(fr.id_list, fr.type_list, fr.box2d_list)
        c2.add(out, data, first=0)
        outs.append(c2.finalize())
    assert outs[0].keys() == outs[1].keys()
    for i in outs[0]:
        assert outs[0][i].keys() == outs[1][i].keys()
        for c in outs[0][i]:
            assert np.array_equal(outs[0][i][c], outs[1][i][c]), (i, c)

