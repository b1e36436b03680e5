"""GPU: the SUN-RGBD evaluator on the device (csrc/sunrgbd_eval.cu via frustum_convnet_b200/sunrgbd_eval.py) against
the reference's own eval_det_cls output (tests/golden/sunrgbd_eval.npz) and against oracle/sunrgbd_eval.py on random
scenes with tied scores, on DetectionCollector output and on a validation-size set.  rec / prec bit-identical, AP
within 1e-12, the logged lines equal; bit-identical results across calls and streams."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(ROOT, "scripts"))


def _compare(res, want_rec, want_prec, want_ap, lines=None):
    for c in want_ap:
        assert np.array_equal(res.rec[c], want_rec[c]), c
        assert np.array_equal(res.prec[c], want_prec[c]), c
        assert abs(res.ap[c] - want_ap[c]) <= 1e-12, (c, res.ap[c], want_ap[c])
    assert sorted(res.ap) == sorted(want_ap)
    if lines is not None:
        assert res.lines() == lines


def _oracle(det_results, gt_rows, gt_ids, classes):
    from oracle import sunrgbd_eval as ose
    r = ose.evaluate(ose.gather_rows(det_results, classes), ose.gt_from_rows(gt_rows, gt_ids))
    return r["rec"], r["prec"], r["ap"], r["lines"]


def _gt(gt_rows, gt_ids, classes, **kw):
    from frustum_convnet_b200.sunrgbd_eval import SunrgbdGroundTruth, gt_corners
    return SunrgbdGroundTruth({c: (gt_corners(gt_rows[c]), gt_ids[c]) for c in classes}, **kw)


@pytest.mark.parametrize("run", ["synth", "real"])
def test_fixture_matches_the_reference(run, tmp_path):
    from frustum_convnet_b200.sunrgbd_eval import SunrgbdEvaluator, SunrgbdGroundTruth
    from test_sunrgbd_eval_cpu import fixture, write_gt_dir
    classes, rows, ids, det, pred_all, want, lines = fixture(run)
    rec = {c: w[0] for c, w in want.items()}
    prec = {c: w[1] for c, w in want.items()}
    ap = {c: w[2] for c, w in want.items()}
    ev = SunrgbdEvaluator(SunrgbdGroundTruth.from_gt_dir(write_gt_dir(tmp_path, run), classes=classes))
    _compare(ev.evaluate(det), rec, prec, ap, lines)
    _compare(ev.evaluate_corners(pred_all), rec, prec, ap, lines)
    _compare(SunrgbdEvaluator(_gt(rows, ids, classes)).evaluate(det), rec, prec, ap, lines)
    res = ev.evaluate(det)
    assert all(res.npos[c] == len(rows[c]) for c in classes)
    if run == "synth":
        assert res.nd["chair"] == 0 and res.ap["chair"] == 0.0 and len(res.rec["chair"]) == 0


@pytest.mark.parametrize("seed", [31, 32, 33])
def test_random_scenes_with_ties_match_the_oracle(seed):
    from frustum_convnet_b200.sunrgbd_eval import SunrgbdEvaluator
    from oracle import sunrgbd_synth as ss
    classes = ("bed", "table", "chair")
    rows, ids, det = ss.make_set(seed, 60, classes, fp_rate=2.0)
    rng = np.random.default_rng(seed)
    for by in det.values():                 # scores on a coarse grid: many ties, decided by gather order
        for d in by.values():
            d[:, 11] = np.round(d[:, 11] * 4) / 4
            d[rng.random(len(d)) < 0.1, 11] = np.float32(-0.0)
    n_ties = sum(len(v) - len(np.unique(v)) for v in
                 ([r[11] for by in det.values() for r in by.get(c, [])] for c in classes))
    assert n_ties > 50
    rec, prec, ap, lines = _oracle(det, rows, ids, classes)
    res = SunrgbdEvaluator(_gt(rows, ids, classes)).evaluate(det)
    _compare(res, rec, prec, ap, lines)


def _collector_output():
    """DetectionCollector(dataset="SUNRGBD").finalize() on the captured reference batches of detect_sunrgbd.npz."""
    from frustum_convnet_b200.detect import DetectionCollector
    from oracle.make_golden_detect import batches
    g = dict(np.load(os.path.join(ROOT, "tests", "golden", "detect_sunrgbd.npz")))
    ids, types = [int(i) for i in g["id_list"]], [str(t) for t in g["type_list"]]
    col = DetectionCollector(ids, types, g["box2d"], dataset="SUNRGBD", method="nms", thresh=float(g["thresh"]))
    for first, outs, rot, rgb, _ in batches(g, False, True):
        d = {"rot_angle": torch.from_numpy(np.asarray(rot).reshape(-1, 1).copy()).cuda(),
             "rgb_prob": torch.from_numpy(np.asarray(rgb).reshape(-1, 1).copy()).cuda()}
        col.add(tuple(torch.from_numpy(np.ascontiguousarray(o)).cuda() for o in outs), d, first=first)
    return col.finalize()


def test_collector_output_end_to_end_matches_the_oracle():
    from frustum_convnet_b200.sunrgbd_eval import CLASS_NAMES, SunrgbdEvaluator
    from oracle import sunrgbd_synth as ss
    det = _collector_output()
    rng = np.random.default_rng(5)
    rows = {c: [] for c in CLASS_NAMES}
    ids = {c: [] for c in CLASS_NAMES}
    for idx, by in det.items():
        for c, d in by.items():
            for k, r in enumerate(np.asarray(d, np.float32).reshape(-1, 12)):
                if k % 3 == 2:
                    continue                                   # a false positive
                p = ss.jitter(rng, r[4:11].astype(np.float64), 0.3, 0.2, 0.3)
                rows[c].append(ss.gt_row(p, rng.random() < 0.5))
                ids[c].append(idx)
    rows[CLASS_NAMES[-1]].append(ss.gt_row(np.array([0, 0, 3, 1, 1, 1, 0.0]), False))   # an image without detections
    ids[CLASS_NAMES[-1]].append(10 ** 6)
    rows = {c: np.asarray(v, np.float64).reshape(-1, 10) for c, v in rows.items()}
    ids = {c: np.asarray(v, np.int64) for c, v in ids.items()}
    rec, prec, ap, lines = _oracle(det, rows, ids, CLASS_NAMES)
    res = SunrgbdEvaluator(_gt(rows, ids, CLASS_NAMES)).evaluate(det)
    _compare(res, rec, prec, ap, lines)
    assert sum(res.nd.values()) > 0 and any(v > 0 for v in res.ap.values())


def test_bit_identical_across_calls_and_streams():
    from frustum_convnet_b200.sunrgbd_eval import CLASS_NAMES, SunrgbdEvaluator
    from oracle import sunrgbd_synth as ss
    rows, ids, det = ss.make_set(7, 400, CLASS_NAMES, check_margins=False, gt_mean=0.5, fp_rate=2.0)
    ev = SunrgbdEvaluator(_gt(rows, ids, CLASS_NAMES))
    key = lambda r: (tuple(r.ap.values()), b"".join(r.rec[c].tobytes() + r.prec[c].tobytes() for c in CLASS_NAMES))
    a, b = key(ev.evaluate(det)), key(ev.evaluate(det))
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    c, d = key(ev.evaluate(det, stream=s1)), key(ev.evaluate(det, stream=s2))
    assert a == b == c == d


def test_validation_size_set_matches_the_oracle():
    from bench_sunrgbd_eval import ground_truth, make_bench_set
    from frustum_convnet_b200.sunrgbd_eval import CLASS_NAMES, SunrgbdEvaluator
    rows, ids, det = make_bench_set()
    assert 15000 < sum(len(r) for r in rows.values()) < 20000
    assert sum(len(v) for by in det.values() for v in by.values()) > 140000
    rec, prec, ap, lines = _oracle(det, rows, ids, CLASS_NAMES)
    res = SunrgbdEvaluator(ground_truth(rows, ids, torch.device("cuda", torch.cuda.current_device()))).evaluate(det)
    _compare(res, rec, prec, ap, lines)


def test_input_validation():
    from frustum_convnet_b200.sunrgbd_eval import SunrgbdEvaluator
    from oracle import sunrgbd_synth as ss
    rows, ids, det = ss.make_set(3, 10, ("bed",), check_margins=False)
    ev = SunrgbdEvaluator(_gt(rows, ids, ("bed",), image_ids=[999]))
    k = next(iter(det))
    bad = {k: {"bed": det[k]["bed"].copy()}}
    bad[k]["bed"][0, 11] = np.nan
    with pytest.raises(ValueError):
        ev.evaluate(bad)
    with pytest.raises(KeyError):
        ev.evaluate({12345: {"bed": det[k]["bed"]}})
    with pytest.raises(ValueError):
        ev.evaluate({2.5: {"bed": det[k]["bed"]}})
    known = float(ids["bed"][0])                         # an integral float id of the ground truth
    r = ev.evaluate({999: {"bed": det[k]["bed"]}, known: {"sofa": det[k]["bed"]}})   # FPs only; sofa ignored
    assert r.nd["bed"] == len(det[k]["bed"]) and r.ap["bed"] == 0.0 and list(r.ap) == ["bed"]
    open_ev = SunrgbdEvaluator(_gt(rows, ids, ("bed",)))  # no id map: any integral id counts, as in the reference
    assert open_ev.evaluate({12345: {"bed": det[k]["bed"]}}).nd["bed"] == len(det[k]["bed"])
