"""Writes tests/golden/sunrgbd_eval.npz: seeded SUN-RGBD evaluation scenes (oracle/sunrgbd_synth.py) and what the
reference's own, unmodified eval_det_cls / get_gt_cls / compute_box_3d make of them.  Needs the reference tree
(oracle/ref_import.REF); the tests read only the fixture.

    python -m oracle.make_golden_sunrgbd_eval               # the fixture
    python -m oracle.make_golden_sunrgbd_eval --time-bench  # eval_det_cls's wall time on scripts/bench_sunrgbd_eval.py's set

Two shims stand in for what the reference imports and this tree lacks: ops.pybind11.box_ops_cc.rbbox_iou_3d_pair is
the float64 oracle/box_iou.py (Boost.Geometry is not available, so Boost parity of the polygon clip stays unpinned,
as in oracle/box_iou.py), and matplotlib / matplotlib.pyplot are no-op stubs (eval_det_cls draws nothing).

Runs (prefix in the file):
  synth  200 images, classes bed, table, sofa, chair, ground truth written as .dat text with both ring orientations;
         chair has ground truth and no detection (the documented divergence: AP 0, empty curves; the reference call
         is skipped for it);
  real   the ground-truth rows of 300 val images of all 10 classes (data only), with jittered detections.
The oracle (oracle/sunrgbd_eval.py) must reproduce the reference's rec / prec bit for bit and its AP within 1e-15.
"""
from __future__ import annotations

import argparse
import os
import sys
import tempfile
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import box_iou  # noqa: E402
from oracle import ref_import  # noqa: E402
from oracle import sunrgbd_eval as ose  # noqa: E402
from oracle import sunrgbd_synth as ss  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "sunrgbd_eval.npz")
GT_DIR = os.path.join(ref_import.REF, "train", "sunrgbd_eval", "gt_boxes")
SYNTH_CLASSES = ("bed", "table", "sofa", "chair")


def reference():
    """-> (eval_det_cls, compare_matlab_python_eval module, compute_box_3d) of the unmodified reference."""
    ref_import._install_shims()
    sys.modules["ops.pybind11.box_ops_cc"].rbbox_iou_3d_pair = box_iou.rbbox_iou_3d_pair
    mpl = types.ModuleType("matplotlib")
    mpl.use = mpl.rc = lambda *a, **k: None
    plt = types.ModuleType("matplotlib.pyplot")
    mpl.pyplot = plt
    sys.modules["matplotlib"], sys.modules["matplotlib.pyplot"] = mpl, plt
    train = os.path.join(ref_import.REF, "train")
    if train not in sys.path:
        sys.path.insert(0, train)
    from sunrgbd_eval import compare_matlab_python_eval as cmp  # type: ignore
    from sunrgbd_eval.eval_det import eval_det_cls  # type: ignore
    from datasets.data_utils import compute_box_3d  # type: ignore
    return eval_det_cls, cmp, compute_box_3d


def pred_all_of(det_results, compute_box_3d):
    """write_detection_results (train/test_net_det_sunrgbd.py:85-117), restated around the reference's own
    compute_box_3d: {class: {idx: [(corners, score)]}}."""
    out = {}
    for idx in det_results:
        for class_type, dets in det_results[idx].items():
            dets = np.asarray(dets, dtype=np.float32)
            for row in dets:
                out.setdefault(class_type, {}).setdefault(idx, []).append(
                    (compute_box_3d(row[4:7], row[7:10], row[10]), row[-1]))
    return out


def flatten(det_results):
    """-> (rows (D, 12) float32, image ids (D,), class names (D,)) in dict order."""
    rows, img, cls = [], [], []
    for idx, by_class in det_results.items():
        for c, d in by_class.items():
            rows.append(np.asarray(d, dtype=np.float32).reshape(-1, 12))
            img += [idx] * len(d)
            cls += [c] * len(d)
    return np.concatenate(rows), np.asarray(img, dtype=np.int64), np.asarray(cls)


def count_taken_best(dets, gt):
    """FPs whose best ground truth is taken while another one is above ovthresh (the no-fall-back rule)."""
    conf = np.array([d[2] for d in dets])
    taken, n = {k: [False] * len(v) for k, v in gt.items()}, 0
    for i in np.argsort(-conf, kind="stable"):
        img, box, _ = dets[i]
        ov = [ose.iou3d(box, g) for g in gt.get(img, [])]
        if not ov or max(ov) <= ss.OVTHRESH:
            continue
        j = int(np.argmax(ov))
        if taken[img][j]:
            n += sum(o > ss.OVTHRESH for k, o in enumerate(ov) if k != j) > 0
        taken[img][j] = True
    return n


def make_run(name, classes, gt_rows, gt_ids, det_results, out, ref):
    eval_det_cls, cmp, compute_box_3d = ref
    with tempfile.TemporaryDirectory() as tmp:
        for c in classes:
            with open(os.path.join(tmp, "%s_gt_boxes.dat" % c), "w") as f:
                f.write(ss.dat_text(gt_rows[c]) if name == "synth" else
                        "".join(" ".join(repr(float(v)) for v in r) + "\n" for r in gt_rows[c]))
            with open(os.path.join(tmp, "%s_gt_imgids.txt" % c), "w") as f:
                f.write(ss.ids_text(gt_ids[c]))
        cmp.gt_boxes_dir = tmp + "/"
        ref_gt = {c: cmp.get_gt_cls(c) for c in classes}
        texts = {c: (open(os.path.join(tmp, "%s_gt_boxes.dat" % c)).read(),
                     open(os.path.join(tmp, "%s_gt_imgids.txt" % c)).read()) for c in classes}
    pred_all = pred_all_of(det_results, compute_box_3d)
    gt_o = ose.gt_from_rows(gt_rows, gt_ids)
    mine = ose.evaluate(ose.gather_rows(det_results, classes), gt_o)
    mine_c = ose.evaluate(ose.gather_corners(pred_all, classes), gt_o)
    ap = {}
    n_taken = 0
    for c in classes:
        npos = sum(len(v) for v in ref_gt[c].values())
        assert npos == mine["npos"][c] == len(gt_rows[c])
        if c not in pred_all:
            assert len(mine["rec"][c]) == 0 and mine["ap"][c] == 0.0
            ap[c] = 0.0
            print(name, c, "no detection: AP 0 (the reference raises KeyError)")
            continue
        rec, prec, a = eval_det_cls(pred_all[c], ref_gt[c], 0.25, False)
        for m in (mine, mine_c):
            assert np.array_equal(m["rec"][c], rec) and np.array_equal(m["prec"][c], prec), (name, c)
            assert abs(m["ap"][c] - a) <= 1e-15, (name, c, m["ap"][c], a)
        ap[c] = float(a)
        n_taken += count_taken_best(ose.gather_rows(det_results, classes)[c], gt_o[c])
        print("%s %-12s npos %5d  nd %5d  tp %5d  AP %.6f" % (name, c, npos, len(rec), int(rec[-1] * npos + 0.5), a))
    mean = float(np.mean([ap[c] for c in classes]))
    lines = ["%s: %.5f" % (c, ap[c]) for c in sorted(ap)] + ["mean_AP: %.5f" % mean]
    assert mine["lines"] == lines
    rows, img, cls = flatten(det_results)
    dup = sum(np.array_equal(rows[i, 4:11], rows[i + 1, 4:11]) for i in range(len(rows) - 1))
    no_gt = sum(1 for i, c in zip(img, cls) if int(i) not in gt_o[str(c)])
    gt_no_det = sum(1 for c in classes for i in gt_o[c] if c not in det_results.get(i, {}))
    print(name, "duplicates", dup, "| best taken, other above 0.25:", n_taken, "| detections without ground truth",
          no_gt, "| ground-truth image lists without detection", gt_no_det)
    assert dup > 0 and no_gt > 0 and gt_no_det > 0 and (n_taken > 0 or name != "synth")
    out[name + "_classes"] = np.array(classes)
    out[name + "_gt_dat"] = np.array([texts[c][0] for c in classes])
    out[name + "_gt_ids_txt"] = np.array([texts[c][1] for c in classes])
    out[name + "_gt_rows"] = np.concatenate([gt_rows[c] for c in classes])
    out[name + "_gt_ids"] = np.concatenate([gt_ids[c] for c in classes])
    out[name + "_gt_class_counts"] = np.array([len(gt_rows[c]) for c in classes])
    out[name + "_det_rows"], out[name + "_det_img"], out[name + "_det_cls"] = rows, img, cls
    # the reference's own corners and scores, in gather order of write_detection_results
    out[name + "_ref_corners"] = np.concatenate([np.stack([b for i in pred_all[c] for b, _ in pred_all[c][i]])
                                                 for c in classes if c in pred_all])
    out[name + "_ref_scores"] = np.concatenate([np.array([s for i in pred_all[c] for _, s in pred_all[c][i]])
                                                for c in classes if c in pred_all])
    rec_ref, prec_ref = [], []
    for c in classes:
        rec_ref.append(mine["rec"][c])
        prec_ref.append(mine["prec"][c])
    out[name + "_nd"] = np.array([len(r) for r in rec_ref])
    out[name + "_rec"], out[name + "_prec"] = np.concatenate(rec_ref), np.concatenate(prec_ref)
    out[name + "_ap"] = np.array([ap[c] for c in classes])
    out[name + "_lines"] = np.array(lines)


def real_gt(n_images, seed):
    """The ground truth of `n_images` val images (every class present): rows and ids per class."""
    rows, ids = {}, {}
    for c in ose.CLASS_NAMES:
        rows[c] = np.loadtxt(os.path.join(GT_DIR, "%s_gt_boxes.dat" % c), ndmin=2)
        ids[c] = np.loadtxt(os.path.join(GT_DIR, "%s_gt_imgids.txt" % c), ndmin=1).astype(np.int64)
    rng = np.random.default_rng(seed)
    pick = set()
    for c in ose.CLASS_NAMES:                          # every class has images in the pick
        pick |= set(rng.choice(np.unique(ids[c]), 3, replace=False).tolist())
    every = np.unique(np.concatenate(list(ids.values())))
    rest = rng.permutation(np.setdiff1d(every, list(pick)))
    pick = sorted(pick | set(rest[:n_images - len(pick)].tolist()))
    sel = {c: np.isin(ids[c], pick) for c in ose.CLASS_NAMES}
    return {c: rows[c][sel[c]] for c in rows}, {c: ids[c][sel[c]] for c in ids}, pick


def time_bench(ref):
    eval_det_cls, cmp, compute_box_3d = ref
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import bench_sunrgbd_eval as bs
    gt_rows, gt_ids, det_results = bs.make_bench_set()
    gt_o = ose.gt_from_rows(gt_rows, gt_ids)
    ref_gt = {c: {float(k): v for k, v in g.items()} for c, g in gt_o.items()}   # get_gt_cls keys are floats
    pred_all = pred_all_of(det_results, compute_box_3d)
    print("%d GT boxes, %d detections" % (sum(len(r) for r in gt_rows.values()),
                                          sum(len(v) for by in det_results.values() for v in by.values())), flush=True)
    t0 = time.perf_counter()
    for c in ose.CLASS_NAMES:
        if c in pred_all:
            eval_det_cls(pred_all[c], ref_gt[c], 0.25, False)
    print("eval_det_cls over the 10 classes (Python loop with the float64 S-H shim, not Boost): %.1f s"
          % (time.perf_counter() - t0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--time-bench", action="store_true")
    args = ap.parse_args()
    if not ref_import.reference_available():
        raise SystemExit("the reference tree is missing: %s" % ref_import.REF)
    ref = reference()
    if args.time_bench:
        time_bench(ref)
        return
    out = {}
    ids = list(np.arange(200) * 7 + 3)
    gt_rows, gt_ids, det = ss.make_set(21, len(ids), SYNTH_CLASSES, ids=ids, no_det_classes=("chair",))
    make_run("synth", SYNTH_CLASSES, gt_rows, gt_ids, det, out, ref)
    rows, rid, pick = real_gt(300, 22)
    given = {}
    for c in ose.CLASS_NAMES:
        for r, i in zip(rows[c], rid[c]):
            given.setdefault(int(i), {}).setdefault(c, []).append(ose.gt_box_corners(r))
    _, _, det = ss.make_set(23, len(pick), ose.CLASS_NAMES, ids=pick, gt_given=given, fp_rate=0.3)
    make_run("real", ose.CLASS_NAMES, rows, rid, det, out, ref)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
