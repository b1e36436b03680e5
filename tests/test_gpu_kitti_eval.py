"""GPU: the KITTI evaluator on the device (csrc/kitti_eval.cu via frustum_convnet_b200/kitti_eval.py) against the
reference evaluator's own output (tests/golden/kitti_eval.npz) and against oracle/kitti_eval.py on random scenes and
on DetectionCollector output.  Precision and AOS vectors within 1e-6, the same evaluated (metric, class) pairs, the
printed AP to its digits; bit-identical results across calls and streams."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(GOLDEN_DIR, "kitti_eval.npz")


def _write(tmp, ids, labels, results):
    gt_dir, res_dir = tmp / "label_2", tmp / "result"
    (res_dir / "data").mkdir(parents=True)
    gt_dir.mkdir()
    for i, lab, det in zip(ids, labels, results):
        (gt_dir / ("%06d.txt" % i)).write_text("".join(ln + "\n" for ln in lab))
        (res_dir / "data" / ("%06d.txt" % i)).write_text("".join(ln + "\n" for ln in det))
    return str(gt_dir), str(res_dir)


def _compare(res, ref, atol=1e-6, aos_atol=1e-6):
    """res: KittiEvalResult; ref: oracle.kitti_eval.evaluate output."""
    for m in ("image", "ground", "3d"):
        assert sorted(res.precision[m]) == sorted(ref["precision"][m]), m
        for c, p in ref["precision"][m].items():
            np.testing.assert_allclose(res.precision[m][c], p, rtol=0, atol=atol, err_msg=(m, c))
            np.testing.assert_allclose(res.ap[m][c], ref["ap"][m][c], rtol=0, atol=5e-4, err_msg=(m, c))
            assert np.array_equal(res.n_gt[m][c], ref["n_gt"][m][c])
            assert np.array_equal(res.n_thresholds[m][c], ref["n_thresholds"][m][c])
    assert res.compute_aos == ref["compute_aos"]
    assert sorted(res.aos) == sorted(ref["aos"])
    for c, a in ref["aos"].items():
        np.testing.assert_allclose(res.aos[c], a, rtol=0, atol=aos_atol, err_msg=c)


@pytest.mark.parametrize("run", ["main", "noaos", "full"])
def test_evaluate_dir_matches_the_reference_evaluator(run, tmp_path):
    from frustum_convnet_b200.kitti_eval import KittiEvaluator, KittiGroundTruth
    from test_kitti_eval_cpu import KINDS
    z = np.load(GOLDEN)
    ids = [int(i) for i in z[run + "_ids"]]
    split = lambda s: [ln for ln in s.split("\n") if ln]
    gt_dir, res_dir = _write(tmp_path, ids, [split(s) for s in z[run + "_labels"]],
                             [split(s) for s in z[run + "_results"]])
    gt = KittiGroundTruth.from_label_dir(gt_dir, ids)
    res = KittiEvaluator(gt).evaluate_dir(res_dir)
    names = list(z[run + "_stats_names"])
    for name, st in zip(names, z[run + "_stats"]):
        _, cls, kind = name.split("_", 2)
        key, m = KINDS[kind]
        got = res.aos.get(cls) if key == "aos" else res.precision[m].get(cls)
        assert got is not None, name
        np.testing.assert_allclose(got, st, rtol=0, atol=1e-6, err_msg=name)
    assert sum(len(res.precision[m]) for m in res.precision) + len(res.aos) == len(names)
    if run == "full":                                # the 41-entry threshold cap is reached on the device
        assert max(int(v.max()) for m in res.n_thresholds.values() for v in m.values()) == 41
    want = [ln.split(" AP: ") for ln in z[run + "_lines"]]
    got = [ln.split(" AP: ") for ln in res.lines()]
    assert [w[0] for w in want] == [g[0] for g in got]
    for w, g in zip(want, got):
        np.testing.assert_allclose(np.array(g[1].split(), float), np.array(w[1].split(), float), atol=2e-6)


@pytest.mark.parametrize("seed", [101, 102, 103, 104])
def test_random_scenes_match_the_oracle(seed):
    from frustum_convnet_b200.kitti_eval import KittiEvaluator, KittiGroundTruth
    from oracle import kitti_eval as ok
    from oracle import kitti_synth as ks
    n = 48
    # seed 104: every object has an exact duplicate, the recall reaches 1 and all 41 thresholds exist
    labels, results = ks.make_set(seed, n, check_margins=True, n_obj=int(4 + seed % 5), det_rate=0.8,
                                  dup_all=seed == 104)
    if seed == 102:
        labels[3] = []                                     # no ground truth
        results[4] = []                                    # no detections
    gts = [ks.parse_label_lines(l) for l in labels]
    dets = [ks.parse_result_lines(r) for r in results]
    ref = ok.evaluate(gts, dets)
    gt = KittiGroundTruth(list(range(n)), gts)
    res = KittiEvaluator(gt).evaluate_records(dets)
    _compare(res, ref)
    assert res.lines() == ref["lines"]
    if seed == 104:
        assert max(int(v.max()) for m in res.n_thresholds.values() for v in m.values()) == 41


def _collector_output():
    """DetectionCollector.finalize() on the captured reference batches of tests/golden/detect_kitti.npz."""
    from frustum_convnet_b200.detect import DetectionCollector
    from oracle.make_golden_detect import batches
    g = dict(np.load(os.path.join(GOLDEN_DIR, "detect_kitti.npz")))
    ids, types = [int(i) for i in g["id_list"]], [str(t) for t in g["type_list"]]
    col = DetectionCollector(ids, types, g["box2d"], dataset="KITTI", method="nms", thresh=float(g["thresh"]))
    for first, outs, rot, rgb, ref in batches(g, False, False):
        d = {"rot_angle": torch.from_numpy(np.asarray(rot).reshape(-1, 1).copy()).cuda()}
        if rgb is not None:
            d["rgb_prob"] = torch.from_numpy(np.asarray(rgb).reshape(-1, 1).copy()).cuda()
        col.add(tuple(torch.from_numpy(np.ascontiguousarray(o)).cuda() for o in outs), d, first=first)
    return col.finalize()


def _compute_alpha(x, z, ry):
    """datasets/provider_sample.py:389-394, restated here: on the float32 scalars of a row, as test() hands them."""
    beta = np.arctan2(z, x)
    alpha = -np.sign(beta) * np.pi / 2 + beta + ry
    return alpha


def _reference_lines(det_results):
    """The text write_detection_results writes (train/test_net_det.py:88-123), per image."""
    out = {}
    for idx in det_results:
        for class_type, dets in det_results[idx].items():
            for row in dets:
                box2d = row[:4]
                tx, ty, tz, h, w, l, ry = row[4:-1]
                alpha = _compute_alpha(tx, tz, ry)
                out.setdefault(idx, []).append(
                    class_type + " -1 -1 " + "%.4f " % alpha + "%.4f %.4f %.4f %.4f " % tuple(box2d) +
                    "%.4f %.4f %.4f %.4f %.4f %.4f %.4f %f" % (h, w, l, tx, ty, tz, ry, row[-1]))
    return out


def test_collector_rows_end_to_end_match_the_oracle_on_the_written_text():
    from frustum_convnet_b200.kitti_eval import KittiEvaluator, KittiGroundTruth
    from oracle import kitti_eval as ok
    from oracle import kitti_synth as ks
    det_results = _collector_output()
    rng = np.random.default_rng(7)
    ids = sorted(int(i) for i in det_results) + [10 ** 6]          # one image without detections
    labels = []
    for idx in ids:
        lab = []
        for class_type, dets in det_results.get(idx, {}).items():
            for k, r in enumerate(dets):
                if k % 3 == 2:
                    continue                                       # a false positive
                x1, y1, x2, y2, tx, ty, tz, h, w, l, ry, _ = (float(v) for v in r)
                sl = rng.uniform(-0.3, 0.3)                        # slid along x: IoUs on both sides of 0.7 / 0.5
                lab.append("%s %.2f %d %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f" % (
                    class_type, rng.choice([0.0, 0.2, 0.4]), rng.integers(0, 3), rng.uniform(-3, 3),
                    x1 + sl * (x2 - x1), y1, x2 + sl * (x2 - x1), y2, h, w, l, tx + sl * l, ty, tz, ry))
        labels.append(lab)
    gts = [ks.parse_label_lines(l) for l in labels]
    text = _reference_lines(det_results)
    dets = [ks.parse_result_lines(text.get(i, [])) for i in ids]
    ref = ok.evaluate(gts, dets)
    res = KittiEvaluator(KittiGroundTruth(ids, gts)).evaluate(det_results)
    # alpha may differ by one unit in the 4th decimal (vectorised against scalar float32 atan2)
    _compare(res, ref, atol=1e-6, aos_atol=1e-5)
    assert any(len(v) for v in res.precision.values())


def test_bit_identical_across_calls_and_streams():
    from frustum_convnet_b200.kitti_eval import KittiEvaluator, KittiGroundTruth
    from oracle import kitti_synth as ks
    labels, results = ks.make_set(5, 300, n_obj=8, det_rate=0.8)
    gts = [ks.parse_label_lines(l) for l in labels]
    dets = [ks.parse_result_lines(r) for r in results]
    ev = KittiEvaluator(KittiGroundTruth(list(range(len(gts))), gts))
    a = bytes(ev.evaluate_records(dets).raw)
    b = bytes(ev.evaluate_records(dets).raw)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    c = bytes(ev.evaluate_records(dets, stream=s1).raw)
    d = bytes(ev.evaluate_records(dets, stream=s2).raw)
    assert a == b == c == d


def test_cpu_tensors_raise():
    from frustum_convnet_b200.kitti_eval import KittiGroundTruth
    with pytest.raises(RuntimeError):
        KittiGroundTruth([1], [np.zeros((0, 15))], device="cpu")
