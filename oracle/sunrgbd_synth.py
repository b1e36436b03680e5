"""TEST INFRASTRUCTURE ONLY - seeded SUN-RGBD evaluation scenes: ground-truth rows as the '<class>_gt_boxes.dat' /
'<class>_gt_imgids.txt' text holds them, and detection dicts {idx: {class: float32 (n, 12)}} slid, scaled and turned
off the ground truth.

Scenes hold both ring orientations, exact duplicate detections (the second is an FP: its ground truth is taken), pairs
where a detection's best ground truth is taken while another one is above the threshold, detections in images
without ground truth of their class and ground-truth images without detections.  ``margins_ok`` keeps every overlap at
least 1e-6 from ovthresh and a detection's two best overlaps identical or 1e-9 apart, so no decision depends on the
last bits in which Boost.Geometry, numpy and the device compute an area (the idea of kitti_synth.margins_ok)."""
from __future__ import annotations

import numpy as np

from . import sunrgbd_eval as ose

OVTHRESH = 0.25


def _params(rng, n):
    """(n, 7) box parameters tx, ty, tz, l, w, h, ry in camera axes."""
    return np.stack([rng.uniform(-3, 3, n), rng.uniform(-0.5, 1.0, n), rng.uniform(1, 7, n), rng.uniform(0.5, 2.5, n),
                     rng.uniform(0.4, 2.0, n), rng.uniform(0.4, 2.0, n), rng.uniform(-np.pi, np.pi, n)], 1)


def gt_row(p, ccw):
    """Box parameters -> one ground-truth row: the (x, z) ring of the box's corners 0-3 (clockwise in the reference's
    sense; reversed when `ccw`), zmin = -(ty + h/2), zmax = -(ty - h/2), rounded as the text holds it."""
    tx, ty, tz, l, w, h, ry = p
    c, s = np.cos(ry), np.sin(ry)
    dx, dz = np.array([l, l, -l, -l]) / 2, np.array([w, -w, -w, w]) / 2
    ring = np.stack([c * dx + s * dz + tx, -s * dx + c * dz + tz], 1)
    if ccw:
        ring = ring[::-1]
    return np.array([float("%.5f" % v) for v in list(ring.reshape(-1)) + [-(ty + h / 2), -(ty - h / 2)]])


def params_of_gt(corners):
    """(8, 3) ground-truth corners -> box parameters whose compute_box_3d corners 0-3 are corners 0-3."""
    p0, p1, p2 = corners[0, [0, 2]], corners[1, [0, 2]], corners[2, [0, 2]]
    w, l = np.hypot(*(p0 - p1)), np.hypot(*(p1 - p2))
    ry = np.arctan2(p0[0] - p1[0], p0[1] - p1[1])
    cen = corners[:4, [0, 2]].mean(0)
    ty, h = (corners[0, 1] + corners[4, 1]) / 2, corners[0, 1] - corners[4, 1]
    return np.array([cen[0], ty, cen[1], l, w, h, ry])


def jitter(rng, p, slide=0.35, scale=0.25, turn=0.4):
    tx, ty, tz, l, w, h, ry = p
    a, b = rng.uniform(-slide, slide, 2)
    c, s = np.cos(ry), np.sin(ry)
    tx, tz = tx + c * a * l + s * b * w, tz - s * a * l + c * b * w
    k = rng.uniform(1 - scale, 1 + scale, 3)
    return np.array([tx, ty + rng.uniform(-0.2, 0.2) * h, tz, l * k[0], w * k[1], h * k[2],
                     ry + rng.uniform(-turn, turn)])


def slide(p, f):
    """p moved by f * l along its heading."""
    q = p.copy()
    q[0] += np.cos(p[6]) * f * p[3]
    q[2] -= np.sin(p[6]) * f * p[3]
    return q


def det_row(p, score):
    return np.concatenate([[0, 0, 0, 0], p, [score]]).astype(np.float32)


def image_scene(rng, classes, n_gt_max=3, fp_rate=1.0, det_classes=None, gt_given=None, gt_mean=None):
    """-> ({class: [(10,) rows]}, {class: [(12,) float32 rows]}) for one image: per class 0..n_gt_max ground-truth
    boxes (Poisson(gt_mean) when given) and Poisson(fp_rate) false positives.  `gt_given`: {class: [(8, 3) corners]}
    of real ground truth to detect instead of drawing boxes."""
    det_classes = classes if det_classes is None else det_classes
    gts, dets = {}, {}
    for c in classes:
        if gt_given is not None:
            ps = [params_of_gt(g) for g in gt_given.get(c, [])]
            rows = []
        else:
            n = int(rng.poisson(gt_mean)) if gt_mean is not None else int(rng.integers(0, n_gt_max + 1))
            ps = list(_params(rng, n))
            if n and rng.random() < 0.3:                       # an overlapping neighbour: best taken, second > 0.25
                ps.append(slide(ps[0], 0.3))
            rows = [gt_row(p, rng.random() < 0.5) for p in ps]
            ps = [params_of_gt(ose.gt_box_corners(r)) for r in rows]
        if rows:
            gts[c] = rows
        if c not in det_classes:
            continue
        d = []
        for k, p in enumerate(ps):
            u = rng.random()
            if u < 0.65:
                d.append(det_row(jitter(rng, p), rng.random()))
            elif u < 0.8:                                       # exact duplicates: the second is an FP
                r = det_row(jitter(rng, p, 0.1, 0.1, 0.1), rng.random())
                d += [r, r.copy()]
                d[-1][11] = r[11] * np.float32(0.5)
            if k == len(ps) - 1 and len(ps) >= 2 and gt_given is None and rng.random() < 0.5:
                d.append(det_row(ps[0], 0.999 - rng.random() * 1e-3))          # takes ps[0]
                d.append(det_row(slide(ps[0], 0.1), rng.random() * 0.5))      # best ps[0] (taken), neighbour > 0.25
        for _ in range(rng.poisson(fp_rate)):
            d.append(det_row(_params(rng, 1)[0], rng.random()))
        if d:
            dets[c] = np.stack(d)
    return gts, dets


def margins_ok(gt_corners, dets):
    """gt_corners {class: [(8, 3)]}, dets {class: (n, 12)} of one image -> every overlap at least 1e-6 from ovthresh
    and the two best overlaps of a detection identical or at least 1e-9 apart."""
    for c, rows in dets.items():
        gs = gt_corners.get(c, [])
        for r in rows:
            b = ose.det_box_corners(r)
            ov = sorted((ose.iou3d(b, g) for g in gs), reverse=True)
            if any(abs(o - OVTHRESH) < 1e-6 for o in ov):
                return False
            if len(ov) >= 2 and ov[0] != ov[1] and ov[0] - ov[1] < 1e-9:
                return False
    return True


def _distinct_scores(det_results, classes):
    for c in classes:
        s = [r[11] for by in det_results.values() for r in by.get(c, [])]
        if len(set(np.float32(s).tolist())) != len(s):
            return False
    return True


def make_set(seed, n_images, classes, ids=None, check_margins=True, no_det_classes=(), gt_given=None, **kw):
    """-> (gt_rows {class: (n, 10)}, gt_ids {class: (n,) int}, det_results {idx: {class: float32 (n, 12)}}).
    `gt_given`: {idx: {class: [(8, 3) corners]}} real ground truth (gt_rows / gt_ids are then empty)."""
    rng = np.random.default_rng(seed)
    ids = list(range(1, n_images + 1)) if ids is None else list(ids)
    det_classes = [c for c in classes if c not in no_det_classes]
    while True:
        gt_rows, gt_ids, det_results = {c: [] for c in classes}, {c: [] for c in classes}, {}
        for idx in ids:
            while True:
                given = gt_given.get(idx, {}) if gt_given is not None else None
                gts, dets = image_scene(rng, classes, det_classes=det_classes, gt_given=given, **kw)
                if not check_margins:
                    break
                gc = given if given is not None else {c: [ose.gt_box_corners(r) for r in rs] for c, rs in gts.items()}
                if margins_ok(gc, dets):
                    break
            for c, rs in gts.items():
                gt_rows[c] += rs
                gt_ids[c] += [idx] * len(rs)
            if dets:
                det_results[idx] = dets
        if not check_margins or _distinct_scores(det_results, classes):
            break
    gt_rows = {c: np.asarray(v, dtype=np.float64).reshape(-1, 10) for c, v in gt_rows.items()}
    gt_ids = {c: np.asarray(v, dtype=np.int64) for c, v in gt_ids.items()}
    return gt_rows, gt_ids, det_results


def dat_text(rows):
    """Ground-truth rows as '<class>_gt_boxes.dat' text (each value already holds 5 decimals)."""
    return "".join(" ".join("%.5f" % v for v in r) + "\n" for r in np.asarray(rows).reshape(-1, 10))


def ids_text(ids):
    """Image ids as '<class>_gt_imgids.txt' holds them: one line of integers."""
    return " ".join("%d" % i for i in ids) + "\n"
