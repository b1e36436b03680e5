"""CPU: the KITTI evaluator's float64 restatement (oracle/kitti_eval.py) against the reference binary's own output
(tests/golden/kitti_eval.npz, oracle/make_golden_kitti_eval.py), the text-free quantisation of the detection rows,
and argument validation of the fcn_kitti_eval_* entries (done on the host, before any CUDA call)."""
import ctypes
import os

import numpy as np
import pytest

from conftest import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden", "kitti_eval.npz")
KINDS = {"detection": ("precision", "image"), "detection_ground": ("precision", "ground"),
         "detection_3d": ("precision", "3d"), "orientation": ("aos", None)}


def _records(z, run):
    from oracle import kitti_synth as ks
    gts = [ks.parse_label_lines([ln for ln in s.split("\n") if ln]) for s in z[run + "_labels"]]
    dets = [ks.parse_result_lines([ln for ln in s.split("\n") if ln]) for s in z[run + "_results"]]
    return gts, dets


def stats_of(res_get, name):
    """stats_<class>_<kind> of the evaluator -> the (3, 41) array of a result (res_get(key, metric, class))."""
    _, cls, kind = name.split("_", 2)
    key, m = KINDS[kind]
    return res_get(key, m, cls)


@pytest.mark.parametrize("run", ["main", "noaos", "full"])
def test_oracle_matches_the_reference_evaluator(run):
    from oracle import kitti_eval as ok
    z = np.load(GOLDEN)
    gts, dets = _records(z, run)
    r = ok.evaluate(gts, dets)
    get = lambda key, m, cls: r[key][m].get(cls) if m else r[key].get(cls)
    names = list(z[run + "_stats_names"])
    for name, st in zip(names, z[run + "_stats"]):
        mine = stats_of(get, name)
        assert mine is not None, name
        np.testing.assert_allclose(mine, st, rtol=0, atol=1e-6, err_msg=name)
    # the same set of evaluated (metric, class) pairs: nothing evaluated that the binary skipped
    n_mine = sum(len(r["precision"][m]) for m in ok.METRICS) + len(r["aos"])
    assert n_mine == len(names)
    assert r["lines"] == list(z[run + "_lines"])
    if run == "noaos":
        assert not r["compute_aos"] and "cyclist" not in r["precision"]["image"]
    if run == "full":
        # all 41 recall steps have a threshold somewhere: the high-recall end of getThresholds, its always-taken last
        # score and the last point of the printed AP are pinned by the evaluator's own vectors
        n_thr = {(m, c): v for m in ok.METRICS for c, v in r["n_thresholds"][m].items()}
        assert max(int(v.max()) for v in n_thr.values()) == 41
        full = [(name, st) for name, st in zip(names, z[run + "_stats"]) if st[:, 40].max() > 0]
        assert full, "no stats vector of the evaluator reaches the 41st point"


def test_fixture_holds_exact_duplicates_of_ground_truth():
    """Detections whose 2-D box and 3-D fields equal a ground truth's: identical polygons, all edges collinear."""
    z = np.load(GOLDEN)
    n = 0
    for run in ("main", "noaos", "full"):
        gts, dets = _records(z, run)
        n += sum(1 for g, d in zip(gts, dets) for row in g for r in d if np.array_equal(row[4:15], r[2:13]))
    assert n > 100


def test_quantisation_equals_printf_and_strtod():
    """'%.4f' / '%f' then float() equals rint(double(v) * 10^k) / 10^k for float32 v, exact decimal ties included."""
    from frustum_convnet_b200.kitti_eval import quantize
    rng = np.random.default_rng(0)
    n = 1_000_000
    v = np.concatenate([
        (rng.standard_normal(n // 4) * 10.0 ** rng.uniform(-6, 3, n // 4)),
        rng.uniform(-1000, 1000, n // 4),
        (2 * rng.integers(-2 ** 20, 2 ** 20, n // 8) + 1) / 32.0,      # x * 1e4 ends in .5 exactly: ties
        (2 * rng.integers(-2 ** 20, 2 ** 20, n // 8) + 1) / 128.0,     # x * 1e6 ends in .5 exactly: ties
        rng.uniform(0, 1, n // 4),
    ]).astype(np.float32)
    assert len(v) == n
    q4, q6 = quantize(v, 4), quantize(v, 6)
    ref4 = np.array([float("%.4f" % x) for x in v.tolist()])
    ref6 = np.array([float("%f" % x) for x in v.tolist()])
    assert np.array_equal(q4, ref4)
    assert np.array_equal(q6, ref6)
    ties = v[n // 2: n // 2 + n // 8]
    assert np.all(np.modf(np.abs(ties.astype(np.float64)) * 1e4)[0] == 0.5)


def test_record_layout_follows_write_detection_results():
    """A detection row becomes the record of the line write_detection_results writes (train/test_net_det.py:88-123)."""
    from frustum_convnet_b200.kitti_eval import compute_alpha, detection_records, parse_result_file
    rng = np.random.default_rng(1)
    rows = rng.uniform(-50, 50, (64, 12)).astype(np.float32)
    rows[:, 11] = rng.uniform(0, 1, 64)
    rec = detection_records(rows, "Pedestrian")
    lines = []
    for r in rows:
        box2d, (tx, ty, tz, h, w, l, ry), score = r[:4], r[4:-1], r[-1]
        alpha = compute_alpha(tx, tz, ry)
        lines.append("Pedestrian -1 -1 " + "%.4f " % alpha + "%.4f %.4f %.4f %.4f " % tuple(box2d) +
                     "%.4f %.4f %.4f %.4f %.4f %.4f %.4f %f" % (h, w, l, tx, ty, tz, ry, score))
    import tempfile
    with tempfile.NamedTemporaryFile("w", suffix=".txt", delete=False) as f:
        f.write("\n".join(lines) + "\n")
    try:
        parsed = parse_result_file(f.name)
    finally:
        os.remove(f.name)
    # alpha from the vectorised float32 atan2 may differ from the scalar one by one float32 ulp (4th decimal flip)
    np.testing.assert_array_equal(np.delete(rec, 1, axis=1), np.delete(parsed, 1, axis=1))
    assert np.abs(rec[:, 1] - parsed[:, 1]).max() <= 1e-4 + 1e-12
    assert rec[0, 0] == 1


def test_type_codes_are_case_insensitive():
    from frustum_convnet_b200.kitti_eval import OTHER, type_code
    assert type_code("Car") == type_code("CAR") == type_code("car") == 0
    assert type_code("Person_sitting") == type_code("person_SITTING") == 4
    assert type_code("DontCare") == 5 and type_code("Truck") == type_code("Tram") == OTHER


def _args(n_img=2, gt_off=(0, 1, 3), det_off=(0, 2, 2)):
    from frustum_convnet_b200 import _lib
    keep = [np.asarray(gt_off, np.int32), np.asarray(det_off, np.int32), np.zeros(64, np.float64)]
    a = _lib.KittiEvalArgs()
    a.num_images, a.num_gt, a.num_det = n_img, int(keep[0][-1]), int(keep[1][-1])
    dummy = keep[2].ctypes.data
    a.gt = a.det = a.gt_offsets = a.det_offsets = a.workspace = a.result = dummy
    a.host_gt_offsets, a.host_det_offsets = keep[0].ctypes.data, keep[1].ctypes.data
    a.workspace_bytes = 1 << 40
    return a, keep


def test_argument_validation_without_gpu():
    from frustum_convnet_b200 import _lib
    lib = _lib.load()
    entries = (lib.fcn_kitti_eval_overlaps, lib.fcn_kitti_eval_thresholds, lib.fcn_kitti_eval_statistics)
    for fn in entries:
        assert fn(None, None) == -1
        assert b"NULL args" in lib.fcn_last_error()
    assert lib.fcn_kitti_eval_workspace_bytes(None) == -1

    def expect(mutate, msg):
        a, keep = _args()
        mutate(a, keep)
        assert lib.fcn_kitti_eval_workspace_bytes(ctypes.byref(a)) == -1
        assert msg in lib.fcn_last_error(), lib.fcn_last_error()
        for fn in entries:
            assert fn(ctypes.byref(a), None) == -1
            assert msg in lib.fcn_last_error(), lib.fcn_last_error()

    expect(lambda a, k: setattr(a, "num_images", -1), b"negative count")
    expect(lambda a, k: setattr(a, "num_det", -3), b"negative count")
    expect(lambda a, k: setattr(a, "gt", None), b"NULL pointer")
    expect(lambda a, k: setattr(a, "det_offsets", None), b"NULL pointer")
    expect(lambda a, k: setattr(a, "host_det_offsets", None), b"NULL host offsets")

    def decreasing(a, k):
        k[0][:] = (0, 2, 1)
        a.num_gt = 1
    expect(decreasing, b"must not decrease")

    def not_zero(a, k):
        k[1][0] = 1
    expect(not_zero, b"start at 0")

    def wrong_total(a, k):
        a.num_gt = 5
    expect(wrong_total, b"num_gt and num_det")

    for field in ("workspace", "result"):         # not needed by the size query, required by the three entries
        a, keep = _args()
        setattr(a, field, None)
        for fn in entries:
            assert fn(ctypes.byref(a), None) == -1
            assert b"NULL workspace or result" in lib.fcn_last_error()


def test_cpu_device_raises():
    from frustum_convnet_b200.kitti_eval import KittiGroundTruth
    with pytest.raises(RuntimeError):
        KittiGroundTruth([0], [np.zeros((0, 15))], device="cpu")
