"""TEST INFRASTRUCTURE ONLY - numpy restatement of the SUN-RGBD detection evaluation (train/sunrgbd_eval/eval_det.py
eval_det / eval_det_cls / voc_ap with use_07_metric=False, the ground-truth conversion of
compare_matlab_python_eval.py:15-67 and compute_box_3d of datasets/data_utils.py:44-70), written row by row so that
it shares no code with frustum_convnet_b200/sunrgbd_eval.py.

Decisions it pins, as the device evaluator makes them:
  * ties in score rank by gather order (a stable sort of the negated scores; -0.0 is 0.0);
  * a class with ground truth and no detection has AP 0 and empty curves (the reference raises KeyError there);
  * the overlap is oracle/box_iou.rbbox_iou_3d_pair (float64 Sutherland-Hodgman, degenerate rings score 0).  Its
    parity with Boost.Geometry stays unpinned, as in oracle/box_iou.py; fixtures keep every decision at least 1e-6
    from ovthresh and competing overlaps 1e-9 apart, so no decision depends on the last bits of an area.
"""
from __future__ import annotations

import numpy as np

from .box_iou import rbbox_iou_3d_pair

CLASS_NAMES = ("bed", "table", "sofa", "chair", "toilet", "desk", "dresser", "night_stand", "bookshelf", "bathtub")


def gt_box_corners(row):
    """One ground-truth row (bird's-eye xy x4, zmin, zmax) -> (8, 3) corners in camera axes."""
    row = np.asarray(row, dtype=np.float64)
    ring = [(row[2 * i], row[2 * i + 1]) for i in range(4)]
    twice_cw = sum(ring[i][0] * ring[i - 1][1] - ring[i][1] * ring[i - 1][0] for i in range(4))
    if not twice_cw > 0:                   # counter-clockwise (or flat): reversed, as box_conversion does
        ring = ring[::-1]
    zmin, zmax = row[8], row[9]
    top = [(x, -zmin, y) for x, y in ring]        # after the swap of wrapper: corners 0-3 carry zmin
    bottom = [(x, -zmax, y) for x, y in ring]
    return np.array(top + bottom, dtype=np.float64)


def det_box_corners(row):
    """One float32 detection row [x1,y1,x2,y2, tx,ty,tz, l,w,h, ry, score] -> (8, 3) float64 corners."""
    row = np.asarray(row, dtype=np.float32)
    ang = row[10]
    c, s = float(np.cos(ang)), float(np.sin(ang))       # float32 cos / sin, as np.cos of a float32 scalar
    l, w, h = (float(row[k] / np.float32(2)) for k in (7, 8, 9))
    dx = (l, l, -l, -l, l, l, -l, -l)
    dy = (h, h, h, h, -h, -h, -h, -h)
    dz = (w, -w, -w, w, w, -w, -w, w)
    tx, ty, tz = (float(v) for v in row[4:7])
    return np.array([(c * dx[k] + s * dz[k] + tx, dy[k] + ty, -s * dx[k] + c * dz[k] + tz) for k in range(8)],
                    dtype=np.float64)


def iou3d(a, b):
    return float(rbbox_iou_3d_pair(a[None], b[None])[0, 1])


def voc_ap(rec, prec):
    mrec = np.concatenate(([0.0], rec, [1.0]))
    mpre = np.concatenate(([0.0], prec, [0.0]))
    for i in range(len(mpre) - 1, 0, -1):
        mpre[i - 1] = max(mpre[i - 1], mpre[i])
    idx = np.nonzero(mrec[1:] != mrec[:-1])[0]
    return float(np.sum((mrec[idx + 1] - mrec[idx]) * mpre[idx + 1]))


def eval_class(dets, gt, ovthresh=0.25):
    """dets: [(image id, corners (8, 3), score)] in gather order; gt: {image id: [corners (8, 3)]} ->
    (rec, prec, ap, npos)."""
    npos = sum(len(v) for v in gt.values())
    taken = {k: [False] * len(v) for k, v in gt.items()}
    if not dets:
        return np.zeros(0), np.zeros(0), 0.0, npos
    conf = np.array([d[2] for d in dets], dtype=np.float64) + 0.0
    order = np.argsort(-conf, kind="stable")
    tp = np.zeros(len(dets))
    fp = np.zeros(len(dets))
    for rank, i in enumerate(order):
        img, box, _ = dets[i]
        boxes = gt.get(img, [])
        ovmax, jmax = -np.inf, -1
        for j, g in enumerate(boxes):
            o = iou3d(np.asarray(box, dtype=np.float64), g)
            if o > ovmax:
                ovmax, jmax = o, j
        if ovmax > ovthresh and not taken[img][jmax]:
            tp[rank] = 1.0
            taken[img][jmax] = True
        else:
            fp[rank] = 1.0
    tp, fp = np.cumsum(tp), np.cumsum(fp)
    with np.errstate(divide="ignore", invalid="ignore"):
        rec = tp / float(npos)
    prec = tp / np.maximum(tp + fp, np.finfo(np.float64).eps)
    return rec, prec, voc_ap(rec, prec), npos


def gather_rows(det_results, classes=CLASS_NAMES):
    """{idx: {class: (n, 12)}} -> {class: [(image id, corners, score)]} in write_detection_results' order."""
    out = {c: [] for c in classes}
    for idx, by_class in det_results.items():
        for name, rows in by_class.items():
            if name not in out:
                continue
            for r in np.asarray(rows, dtype=np.float32).reshape(-1, 12):
                out[name].append((int(idx), det_box_corners(r), float(r[11])))
    return out


def gather_corners(pred_all, classes=CLASS_NAMES):
    """{class: {idx: [(corners, score)]}} -> {class: [(image id, corners, score)]}."""
    return {c: [(int(idx), np.asarray(b, dtype=np.float64), float(s)) for idx, lst in pred_all.get(c, {}).items()
                for b, s in lst] for c in classes}


def gt_from_rows(boxes_by_class, ids_by_class):
    """{class: (n, 10) rows}, {class: (n,) ids} -> {class: {image id: [corners]}} in row order."""
    gt = {}
    for c, rows in boxes_by_class.items():
        per = {}
        for row, i in zip(np.asarray(rows).reshape(-1, 10), np.asarray(ids_by_class[c]).reshape(-1)):
            per.setdefault(int(i), []).append(gt_box_corners(row))
        gt[c] = per
    return gt


def evaluate(dets_by_class, gt_by_class, ovthresh=0.25):
    """-> {"rec", "prec", "ap", "npos": {class: ...}, "mean_ap", "lines"} over the classes of the ground truth."""
    out = {"rec": {}, "prec": {}, "ap": {}, "npos": {}}
    for c, gt in gt_by_class.items():
        rec, prec, ap, npos = eval_class(dets_by_class.get(c, []), gt, ovthresh)
        out["rec"][c], out["prec"][c], out["ap"][c], out["npos"][c] = rec, prec, ap, npos
    out["mean_ap"] = float(np.mean([out["ap"][c] for c in out["ap"]]))
    out["lines"] = ["%s: %.5f" % (c, out["ap"][c]) for c in sorted(out["ap"])] + ["mean_AP: %.5f" % out["mean_ap"]]
    return out
