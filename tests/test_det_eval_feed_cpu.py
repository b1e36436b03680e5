"""CPU: the host half of ``evaluate_collected`` (the gather plans of kitti_eval / sunrgbd_eval built from a
collector's segment metadata) against the row order of the dict path, and the device feed's quantization and alpha
restated in numpy float64 against kitti_eval.quantize / compute_alpha.  The plans are applied here by a numpy
restatement of the feed kernels' scatter (csrc/det_eval_feed.cu)."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from frustum_convnet_b200 import kitti_eval as ke
from frustum_convnet_b200 import sunrgbd_eval as se
from frustum_convnet_b200.detect import CollectedDetections


def fake_collected(keys, counted, kept, added, seed=0):
    """A collector's finalized state: segments `keys` (the collector's table order), `counted` rows per segment of
    which the first `kept` are kept, frustum s added when added[s] (one frustum per segment, dataset order = table
    order here).  Row values are unique (column 11 holds the row index)."""
    rng = np.random.default_rng(seed)
    S = len(keys)
    off = np.zeros(S + 1, np.int32)
    np.cumsum(counted, out=off[1:])
    rows = rng.uniform(-5, 5, (int(off[-1]), 12)).astype(np.float32)
    rows[:, 11] = np.arange(len(rows))
    order = np.flatnonzero(np.asarray(added, bool))
    return CollectedDetections("KITTI", torch.from_numpy(rows), None, None, off, np.asarray(kept, np.int32),
                               list(keys), order, None)


def scatter(col, seg_dst, n_out):
    """What the feed kernels do: counted row r of segment s, k < keep_count[s], goes to seg_dst[s] + k."""
    rows = col.rows.numpy()
    out = np.full((n_out, 12), np.nan, np.float32)
    src = np.full(n_out, -1)
    for s in range(col.num_segments):
        a, kc, d = col.host_seg_offsets[s], col.host_keep_count[s], seg_dst[s]
        if d >= 0:
            assert (src[d:d + kc] == -1).all()
            out[d:d + kc], src[d:d + kc] = rows[a:a + kc], s
    assert (src >= 0).all()
    return out, src


# interleaved images and classes, zero-row segments, a non-added frustum, and (for the GT) images outside it
KEYS = [(7, "Car"), (3, "Pedestrian"), (7, "Cyclist"), (3, "Car"), (9, "Car"), (7, "Pedestrian"), (12, "Car"),
        (3, "Cyclist"), (9, "Van"), (5, "Car")]
COUNTED = [5, 3, 0, 4, 2, 6, 1, 3, 2, 4]
KEPT = [3, 2, 0, 4, 0, 5, 1, 2, 1, 4]
ADDED = [1, 1, 1, 1, 1, 1, 1, 1, 1, 0]              # (5, Car) was never added


def _kitti_evaluator(image_ids):
    gt = types.SimpleNamespace(image_ids=list(image_ids), index={i: k for k, i in enumerate(image_ids)}, device=None)
    return ke.KittiEvaluator(gt)


def test_kitti_plan_matches_the_dict_path():
    col = fake_collected(KEYS, COUNTED, KEPT, ADDED)
    ev = _kitti_evaluator([12, 1, 3, 9, 7, 5])
    seg_dst, seg_code, det_off = ev.gather_plan(col)
    out, src = scatter(col, seg_dst, int(det_off[-1]))
    dets = col.to_dict()
    # the dict path's per-image order (KittiEvaluator.evaluate)
    per_image = [[] for _ in ev.gt.image_ids]
    for idx, by_class in dets.items():
        for ct, d in by_class.items():
            if len(d):
                per_image[ev.gt.index[idx]].append((d, ke.type_code(ct)))
    want = np.concatenate([d for p in per_image for d, _ in p])
    assert np.array_equal(out, want)
    assert np.array_equal(np.diff(det_off), [sum(len(d) for d, _ in p) for p in per_image])
    assert np.array_equal(seg_code[src], np.concatenate([np.full(len(d), c) for p in per_image for d, c in p]))
    assert seg_dst[9] == -1                          # not added: no rows written


def test_kitti_plan_raises_for_an_image_outside_the_ground_truth():
    col = fake_collected(KEYS, COUNTED, KEPT, ADDED)
    with pytest.raises(KeyError):
        _kitti_evaluator([12, 3, 7]).gather_plan(col)   # 9 is missing
    _kitti_evaluator([12, 3, 7, 9]).gather_plan(col)    # 5 is missing but was never added


def test_kitti_plan_empty():
    col = fake_collected([], [], [], [])
    seg_dst, _, det_off = _kitti_evaluator([1, 2]).gather_plan(col)
    assert len(seg_dst) == 0 and list(det_off) == [0, 0, 0]


SUN_KEYS = [(4, "chair"), (2, "table"), (4, "table"), (2, "chair"), (6, "lamp"), (8, "table"), (6, "chair"),
            (9, "chair")]
SUN_COUNTED = [3, 2, 4, 0, 2, 3, 1, 2]
SUN_KEPT = [3, 1, 4, 0, 2, 2, 1, 2]
SUN_ADDED = [1, 1, 1, 1, 1, 1, 1, 0]


def _sunrgbd_evaluator(classes, segment_of, known=None):
    gt = types.SimpleNamespace(classes=tuple(classes), class_index={c: i for i, c in enumerate(classes)},
                               segment_of=dict(segment_of), known_images=known, device=None)
    return se.SunrgbdEvaluator(gt)


def test_sunrgbd_plan_matches_the_dict_path():
    col = fake_collected(SUN_KEYS, SUN_COUNTED, SUN_KEPT, SUN_ADDED)
    # classes with ground truth: table, chair (not lamp); (class, image) segments for some images only
    ev = _sunrgbd_evaluator(["table", "chair", "sofa"], {(0, 2): 0, (0, 8): 1, (1, 4): 2, (1, 6): 3})
    seg_dst, seg_gt, det_off = ev.gather_plan(col)
    out, src = scatter(col, seg_dst, int(det_off[-1]))
    dets = col.to_dict()
    # the dict path's gather (SunrgbdEvaluator.evaluate): class after class, images in dict order, then rows
    rows, segs = [[] for _ in ev.gt.classes], [[] for _ in ev.gt.classes]
    for idx, by_class in dets.items():
        for name, d in by_class.items():
            ci = ev.gt.class_index.get(name)
            if ci is not None:
                rows[ci].append(d)
                segs[ci].append(ev._segments(ci, se.image_key(idx), len(d)))
    assert np.array_equal(out, np.concatenate([r for per in rows for r in per]))
    assert np.array_equal(seg_gt[src], np.concatenate([s for per in segs for s in per]))
    assert np.array_equal(np.diff(det_off), [sum(len(r) for r in per) for per in rows])
    # the issue's example: table rows of image 4 (dict position 0) come before those of image 2 (position 1)
    table = out[:det_off[1], 11]
    first_4 = col.host_seg_offsets[2]
    assert table[0] == first_4
    assert seg_dst[4] == -1 and seg_dst[7] == -1     # lamp has no ground truth; (9, chair) was never added


def test_sunrgbd_plan_checks_every_image_of_the_dict():
    col = fake_collected(SUN_KEYS, SUN_COUNTED, SUN_KEPT, SUN_ADDED)
    ev = _sunrgbd_evaluator(["table", "chair"], {(0, 2): 0}, known={2, 4, 8})
    with pytest.raises(KeyError):
        ev.gather_plan(col)                          # image 6 (chair and lamp) is unknown
    _sunrgbd_evaluator(["table", "chair"], {(0, 2): 0}, known={2, 4, 6, 8}).gather_plan(col)


# ------------------------------------------------------------------------------------------ the feed's arithmetic
def device_quantize(v, decimals):
    """csrc/det_eval_feed.cu df_quantize restated: rint(float64(v) * 10^d) / 10^d, ties to even."""
    s = 10.0 ** decimals
    return np.rint(np.asarray(v, np.float32).astype(np.float64) * s) / s


def device_alpha(x, z, ry):
    """df_alpha restated: atan2 in float64 rounded once to float32, then numpy's float32 order."""
    x, z, ry = (np.asarray(v, np.float32) for v in (x, z, ry))
    b = np.arctan2(z.astype(np.float64), x.astype(np.float64)).astype(np.float32)
    t = (-np.sign(b) * np.float32(np.pi)).astype(np.float32) / np.float32(2)
    return ((t + b).astype(np.float32) + ry).astype(np.float32)


def test_quantize_restatement_equals_kitti_eval_quantize():
    rng = np.random.default_rng(3)
    v = np.concatenate([rng.uniform(-100, 100, 200000), rng.uniform(-1, 1, 100000)]).astype(np.float32)
    ties4 = (np.arange(-401, 402, 2) / 32.0).astype(np.float32)          # odd / 32: x * 1e4 = k + 1/2 exactly
    ties6 = (np.arange(-401, 402, 2) / 128.0).astype(np.float32)         # odd / 128: x * 1e6 = k + 1/2 exactly
    assert (ties4.astype(np.float64) * 1e4 % 1 == 0.5).all() and (ties6.astype(np.float64) * 1e6 % 1 == 0.5).all()
    for d, extra in ((4, ties4), (6, ties6)):
        x = np.concatenate([v, extra, np.float32([0.0, -0.0, np.inf, -np.inf])])
        a, b = device_quantize(x, d), ke.quantize(x, d)
        assert np.array_equal(a.view(np.int64), b.view(np.int64))
    assert device_quantize(np.float32(1 / 32), 4) == 0.0312 and device_quantize(np.float32(3 / 32), 4) == 0.0938


def test_alpha_restatement_against_compute_alpha():
    rng = np.random.default_rng(5)
    n = 400000
    x = rng.uniform(-40, 40, n).astype(np.float32)
    z = rng.uniform(-5, 80, n).astype(np.float32)
    ry = rng.uniform(-np.pi, np.pi, n).astype(np.float32)
    x[:50], z[:50] = 0, rng.uniform(1, 5, 50).astype(np.float32)                 # on the axes
    z[50:100] = 0
    dev, host = device_alpha(x, z, ry), ke.compute_alpha(x, z, ry).astype(np.float32)
    b_host = np.arctan2(z, x)
    b_cr = np.arctan2(z.astype(np.float64), x.astype(np.float64)).astype(np.float32)
    same = b_host == b_cr
    # bit-identical wherever numpy's float32 atan2 is the correctly rounded value
    assert np.array_equal(dev[same].view(np.int32), host[same].view(np.int32))
    # within one '%.4f' step after the rounding everywhere
    assert np.abs(device_quantize(dev, 4) - ke.quantize(host, 4)).max() <= 1e-4 + 1e-12
    print("numpy float32 arctan2 differs from the correctly rounded value on %.1f %% of inputs" %
          (100 * (~same).mean()))


def test_feed_symbols_are_declared():
    from frustum_convnet_b200 import _lib
    for name in ("fcn_det_kitti_records", "fcn_det_sunrgbd_feed"):
        assert name in _lib.SIGNATURES


def test_feed_entries_validate_on_the_host():
    """Validation comes before any CUDA call, so it is testable without a GPU."""
    from frustum_convnet_b200 import _lib, build
    build.build()
    lib = _lib.load()
    off = np.array([0, 3, 5], np.int32)
    kc = np.array([2, 2], np.int32)

    def args(dst, num_out, offsets=off, keep=kc, num_rows=5):
        a = _lib.DetEvalFeedArgs()
        a.num_segments, a.num_rows, a.num_out = 2, num_rows, num_out
        a.host_seg_offsets, a.host_keep_count, a.host_seg_dst = offsets.ctypes.data, keep.ctypes.data, dst.ctypes.data
        return a

    for fn in (lib.fcn_det_kitti_records, lib.fcn_det_sunrgbd_feed):
        assert fn(None, None) == -1
        bad = [(np.array([0, 2], np.int32), 3, off, kc, 5, b"num_out"),                 # rows overrun num_out
               (np.array([0, 2], np.int32), 5, off, kc, 5, b"add up"),                  # kept rows != num_out
               (np.array([-2, 0], np.int32), 2, off, kc, 5, b"seg_dst"),
               (np.array([0, 2], np.int32), 4, np.array([0, 3, 4], np.int32), kc, 5, b"seg_offsets"),
               (np.array([0, 2], np.int32), 4, np.array([0, 1, 5], np.int32), kc, 5, b"keep_count")]
        for dst, n_out, o, k, nr, msg in bad:
            assert fn(C.byref(args(dst, n_out, o, k, nr)), None) == -1, msg
            assert msg in lib.fcn_last_error(), lib.fcn_last_error()
        dst = np.array([0, 2], np.int32)
        assert fn(C.byref(args(dst, 4)), None) == -1                                    # valid plan, NULL pointers
        assert b"NULL" in lib.fcn_last_error()

