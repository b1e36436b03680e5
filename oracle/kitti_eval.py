"""TEST INFRASTRUCTURE ONLY - numpy / float64 restatement of the KITTI offline evaluator
(train/kitti_eval/evaluate_object_3d_offline.cpp:56-916), pinned to the reference binary's own output by
tests/test_kitti_eval_cpu.py on tests/golden/kitti_eval.npz (oracle/make_golden_kitti_eval.py).

Inputs are the record layout of include/frustum_b200.h section (13), one float64 array per image:
    gt  (ng, 15) [code, truncation, occlusion, alpha, x1, y1, x2, y2, h, w, l, t1, t2, t3, ry]
    det (nd, 14) [code, alpha, x1, y1, x2, y2, h, w, l, t1, t2, t3, ry, score]
with the type codes of frustum_convnet_b200.kitti_eval.TYPE_CODES.

The functions follow the reference one for one (cleanData, computeStatistics, getThresholds, eval_class,
saveAndPlotPlots' AP line); the only restructuring is that every (detection, ground truth) overlap is computed once
per metric instead of inside every threshold loop.  The bird's-eye-view polygons are toPolygon's (:271-293) and
their intersection is the float64 Sutherland-Hodgman clip of oracle/box_iou.py; the union of two overlapping convex
polygons has the area a + b - inter.  Boost.Geometry's areas differ from these in the last bits only; the fixture
keeps every overlap at least 1e-9 away from its threshold so that no decision depends on them.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import box_iou as ob

CAR, PEDESTRIAN, CYCLIST, VAN, PERSON_SITTING, DONTCARE, OTHER = range(7)
CLASS_NAMES = ("car", "pedestrian", "cyclist")
METRICS = ("image", "ground", "3d")
MIN_HEIGHT = (40, 25, 25)
MAX_OCCLUSION = (0, 1, 2)
MAX_TRUNCATION = (0.15, 0.3, 0.5)
MIN_OVERLAP = ((0.7, 0.5, 0.5), (0.7, 0.5, 0.5), (0.7, 0.5, 0.5))
N_SAMPLE_PTS = 41
NO_DETECTION = -10000000.0

# record columns
G_CODE, G_TRUNC, G_OCCL, G_ALPHA, G_X1, G_Y1, G_X2, G_Y2, G_H, G_W, G_L, G_T1, G_T2, G_T3, G_RY = range(15)
D_CODE, D_ALPHA, D_X1, D_Y1, D_X2, D_Y2, D_H, D_W, D_L, D_T1, D_T2, D_T3, D_RY, D_SCORE = range(14)


# ------------------------------------------------------------------------------------------------ overlaps
def image_overlap(d, g, crit0):
    """imageBoxOverlap (:229-263), a = detection, b = ground truth."""
    x1, y1 = max(d[D_X1], g[G_X1]), max(d[D_Y1], g[G_Y1])
    x2, y2 = min(d[D_X2], g[G_X2]), min(d[D_Y2], g[G_Y2])
    w, h = x2 - x1, y2 - y1
    if w <= 0 or h <= 0:
        return 0.0
    inter = w * h
    a_area = (d[D_X2] - d[D_X1]) * (d[D_Y2] - d[D_Y1])
    b_area = (g[G_X2] - g[G_X1]) * (g[G_Y2] - g[G_Y1])
    return inter / a_area if crit0 else inter / (a_area + b_area - inter)


def polygon(ry, l, w, t1, t3):
    """toPolygon (:271-293): [[c, s], [-s, c]] @ (+-l/2, +-w/2) + (t1, t3), corners in the reference's order."""
    c, s = math.cos(ry), math.sin(ry)
    dx = (l / 2, l / 2, -l / 2, -l / 2)
    dz = (w / 2, -w / 2, -w / 2, w / 2)
    return np.array([[c * dx[i] + s * dz[i] + t1, -s * dx[i] + c * dz[i] + t3] for i in range(4)])


def rotated_overlaps(d, g, crit0):
    """(groundBoxOverlap, box3DOverlap) (:296-346)."""
    gp = polygon(g[G_RY], g[G_L], g[G_W], g[G_T1], g[G_T3])
    dp = polygon(d[D_RY], d[D_L], d[D_W], d[D_T1], d[D_T3])
    inter = ob._clip_convex(gp, dp)
    inter_area = abs(ob._shoelace_ccw(inter)) if len(inter) >= 3 else 0.0
    g_area, d_area = -ob._shoelace_ccw(gp), -ob._shoelace_ccw(dp)
    with np.errstate(divide="ignore", invalid="ignore"):
        bev = np.float64(inter_area) / (d_area if crit0 else g_area + d_area - inter_area)
        ymax = min(d[D_T2], g[G_T2])
        ymin = max(d[D_T2] - d[D_H], g[G_T2] - g[G_H])
        inter_vol = inter_area * max(0.0, ymax - ymin)
        det_vol = d[D_H] * d[D_L] * d[D_W]
        gt_vol = g[G_H] * g[G_L] * g[G_W]
        o3d = np.float64(inter_vol) / (det_vol if crit0 else det_vol + gt_vol - inter_vol)
    return float(bev), float(o3d)


def image_pair_overlaps(gt, det):
    """(3, nd, ng): the overlap of every pair per metric; criterion 0 against DontCare ground truth (:582)."""
    nd, ng = len(det), len(gt)
    ov = np.zeros((3, nd, ng))
    for j in range(nd):
        for k in range(ng):
            crit0 = int(gt[k, G_CODE]) == DONTCARE
            ov[0, j, k] = image_overlap(det[j], gt[k], crit0)
            ov[1, j, k], ov[2, j, k] = rotated_overlaps(det[j], gt[k], crit0)
    return ov


# ------------------------------------------------------------------------------------------------ evaluation
def clean_data(cls, diff, gt, det):
    """cleanData (:383-456) -> ignored_gt, ignored_det, dontcare indices, n_gt."""
    ignored_gt, n_gt = [], 0
    for g in gt:
        code = int(g[G_CODE])
        if code == cls:
            valid = 1
        elif (cls == PEDESTRIAN and code == PERSON_SITTING) or (cls == CAR and code == VAN):
            valid = 0
        else:
            valid = -1
        height = g[G_Y2] - g[G_Y1]
        ignore = int(g[G_OCCL]) > MAX_OCCLUSION[diff] or g[G_TRUNC] > MAX_TRUNCATION[diff] or height < MIN_HEIGHT[diff]
        if valid == 1 and not ignore:
            ignored_gt.append(0)
            n_gt += 1
        elif valid == 0 or (ignore and valid == 1):
            ignored_gt.append(1)
        else:
            ignored_gt.append(-1)
    dc = [k for k in range(len(gt)) if int(gt[k, G_CODE]) == DONTCARE]
    ignored_det = []
    for d in det:
        height = int(abs(d[D_Y1] - d[D_Y2]))                         # int32_t height = fabs(...) (:446)
        if height < MIN_HEIGHT[diff]:
            ignored_det.append(1)
        elif int(d[D_CODE]) == cls:
            ignored_det.append(0)
        else:
            ignored_det.append(-1)
    return ignored_gt, ignored_det, dc, n_gt


def compute_statistics(m, cls, gt, det, ov, dc, ignored_gt, ignored_det, compute_fp, compute_aos=False, thresh=0.0):
    """computeStatistics (:458-616); ov = this image's (nd, ng) overlaps of metric m.
    -> (tp, fp, fn, similarity, tp scores)."""
    min_overlap = MIN_OVERLAP[m][cls]
    nd = len(det)
    assigned = [False] * nd
    ignored_threshold = [compute_fp and det[j, D_SCORE] < thresh for j in range(nd)]
    tp = fp = fn = 0
    v, delta = [], []
    for i in range(len(gt)):
        if ignored_gt[i] == -1:
            continue
        det_idx, valid_detection, max_overlap, assigned_ignored_det = -1, NO_DETECTION, 0.0, False
        for j in range(nd):
            if ignored_det[j] == -1 or assigned[j] or ignored_threshold[j]:
                continue
            overlap = ov[j, i]
            if not compute_fp and overlap > min_overlap and det[j, D_SCORE] > valid_detection:
                det_idx, valid_detection = j, det[j, D_SCORE]
            elif (compute_fp and overlap > min_overlap and (overlap > max_overlap or assigned_ignored_det)
                  and ignored_det[j] == 0):
                max_overlap, det_idx, valid_detection, assigned_ignored_det = overlap, j, 1.0, False
            elif compute_fp and overlap > min_overlap and valid_detection == NO_DETECTION and ignored_det[j] == 1:
                det_idx, valid_detection, assigned_ignored_det = j, 1.0, True
        if valid_detection == NO_DETECTION and ignored_gt[i] == 0:
            fn += 1
        elif valid_detection != NO_DETECTION and (ignored_gt[i] == 1 or ignored_det[det_idx] == 1):
            assigned[det_idx] = True
        elif valid_detection != NO_DETECTION:
            tp += 1
            v.append(det[det_idx, D_SCORE])
            if compute_aos:
                delta.append(gt[i, G_ALPHA] - det[det_idx, D_ALPHA])
            assigned[det_idx] = True
    similarity = 0.0
    if compute_fp:
        for j in range(nd):
            if not (assigned[j] or ignored_det[j] == -1 or ignored_det[j] == 1 or ignored_threshold[j]):
                fp += 1
        nstuff = 0
        for k in dc:
            for j in range(nd):
                if assigned[j] or ignored_det[j] in (-1, 1) or ignored_threshold[j]:
                    continue
                if ov[j, k] > min_overlap:
                    assigned[j] = True
                    nstuff += 1
        fp -= nstuff
        if compute_aos:
            if tp > 0 or fp > 0:
                similarity = 0.0
                for dl in delta:
                    similarity += (1.0 + math.cos(dl)) / 2.0
            else:
                similarity = -1.0
    return tp, fp, fn, similarity, v


def get_thresholds(v, n_groundtruth):
    """getThresholds (:348-381)."""
    v = sorted(v, reverse=True)
    t = []
    current_recall = 0.0
    for i in range(len(v)):
        l_recall = (i + 1) / float(n_groundtruth)
        r_recall = (i + 2) / float(n_groundtruth) if i < len(v) - 1 else l_recall
        if (r_recall - current_recall) < (current_recall - l_recall) and i < len(v) - 1:
            continue
        t.append(v[i])
        current_recall += 1.0 / (N_SAMPLE_PTS - 1.0)
    return t


def _suffix_max(x, i):
    """*std::max_element(x.begin() + i, x.end()): the first element no later one exceeds."""
    best = i
    for k in range(i + 1, len(x)):
        if x[best] < x[k]:
            best = k
    return x[best]


def eval_class(m, cls, diff, gts, dets, ovs, compute_aos):
    """eval_class (:622-704) -> (precision (41,), aos (41,) or None, number of thresholds, n_gt)."""
    n_gt, v, cleaned = 0, [], []
    for gt, det, ov in zip(gts, dets, ovs):
        ig, idt, dc, n = clean_data(cls, diff, gt, det)
        n_gt += n
        cleaned.append((ig, idt, dc))
        v += compute_statistics(m, cls, gt, det, ov[m], dc, ig, idt, False)[4]
    thresholds = get_thresholds(v, n_gt)
    T = len(thresholds)
    tp, fp, sim = [0] * T, [0] * T, [0.0] * T
    for (gt, det, ov), (ig, idt, dc) in zip(zip(gts, dets, ovs), cleaned):
        for t in range(T):
            a, b, _, s, _ = compute_statistics(m, cls, gt, det, ov[m], dc, ig, idt, True, compute_aos, thresholds[t])
            tp[t] += a
            fp[t] += b
            if s != -1:
                sim[t] += s
    precision = [0.0] * N_SAMPLE_PTS
    aos = [0.0] * N_SAMPLE_PTS if compute_aos else None
    with np.errstate(divide="ignore", invalid="ignore"):
        for i in range(T):
            precision[i] = float(np.float64(tp[i]) / np.float64(tp[i] + fp[i]))
            if compute_aos:
                aos[i] = float(np.float64(sim[i]) / np.float64(tp[i] + fp[i]))
    for i in range(T):
        precision[i] = _suffix_max(precision, i)
        if compute_aos:
            aos[i] = _suffix_max(aos, i)
    return np.array(precision), (np.array(aos) if compute_aos else None), T, n_gt


def printed_ap(vals):
    """saveAndPlotPlots' AP (:716-720): float32 sum (float += double) of steps 0, 4, ..., 40, / 11 * 100."""
    s = np.float32(0)
    for i in range(0, len(vals), 4):
        s = np.float32(np.float64(s) + vals[i])
    return float(s / np.float32(11) * np.float32(100))


def run_flags(dets):
    """loadDetections (:157-172): per class eval_image / eval_ground / eval_3d, and compute_aos."""
    flags = np.zeros((3, 3), dtype=bool)
    compute_aos = True
    for det in dets:
        for d in det:
            if d[D_ALPHA] == -10:
                compute_aos = False
            c = int(d[D_CODE])
            if c > 2:
                continue
            flags[0, c] |= d[D_X1] >= 0
            flags[1, c] |= d[D_T1] != -1000
            flags[2, c] |= d[D_T2] != -1000
    return flags, compute_aos


def evaluate(gts, dets):
    """The whole run (eval, :792-916).  -> dict with
        precision[metric][class] (3, 41), aos[class] (3, 41), ap[metric][class] (3,), ap_aos[class] (3,),
        n_thresholds[metric][class] (3,), n_gt[metric][class] (3,), compute_aos, lines (the printed AP lines)
    holding only the evaluated classes (a class without a detection that enables the metric is absent)."""
    flags, compute_aos = run_flags(dets)
    ovs = [image_pair_overlaps(np.asarray(g, np.float64).reshape(-1, 15), np.asarray(d, np.float64).reshape(-1, 14))
           for g, d in zip(gts, dets)]
    gts = [np.asarray(g, np.float64).reshape(-1, 15) for g in gts]
    dets = [np.asarray(d, np.float64).reshape(-1, 14) for d in dets]
    out = {k: {m: {} for m in METRICS} for k in ("precision", "ap", "n_thresholds", "n_gt")}
    out.update(aos={}, ap_aos={}, compute_aos=compute_aos, lines=[])
    suffix = ("_detection", "_detection_ground", "_detection_3d")
    for m in range(3):
        for c in range(3):
            if not flags[m, c]:
                continue
            aos_m = compute_aos and m == 0
            res = [eval_class(m, c, d, gts, dets, ovs, aos_m) for d in range(3)]
            name = CLASS_NAMES[c]
            out["precision"][METRICS[m]][name] = np.stack([r[0] for r in res])
            out["n_thresholds"][METRICS[m]][name] = np.array([r[2] for r in res])
            out["n_gt"][METRICS[m]][name] = np.array([r[3] for r in res])
            ap = np.array([printed_ap(r[0]) for r in res])
            out["ap"][METRICS[m]][name] = ap
            out["lines"].append("%s AP: %f %f %f" % ((name + suffix[m],) + tuple(ap)))
            if aos_m:
                out["aos"][name] = np.stack([r[1] for r in res])
                out["ap_aos"][name] = np.array([printed_ap(r[1]) for r in res])
                out["lines"].append("%s AP: %f %f %f" % ((name + "_orientation",) + tuple(out["ap_aos"][name])))
    return out
