"""Seeded synthetic KITTI label and result files for the evaluator's fixtures, tests and benchmark.

``make_scene(rng, ...)`` returns one image as two lists of text lines, a label_2 file and a result file, built from
the families the evaluator branches on:
  * ground truth of every type (Car, Pedestrian, Cyclist, Van, Person_sitting, Truck, DontCare) with truncation,
    occlusion and 2-D heights on and around each difficulty boundary (0.15 / 0.3 / 0.5, 0 / 1 / 2, 40 / 25 px);
  * per object: an exact duplicate (the detection line repeats the label's own printed values, so the 2-D box and the
    bird's-eye-view polygon are identical to the ground truth's), boxes slid along their heading (and turned a
    little) to IoUs on both sides of 0.7 and 0.5, a second detection of the same box (an FP), neighbour-class
    detections (Car on a Van); with ``dup_all`` every object also gets an exact duplicate of its evaluated class, so
    the recall of a class reaches 1 and all 41 recall steps get a threshold;
  * detections with 2-D heights below 25 and 40 px, including fractional heights that int truncation flips;
  * detections inside DontCare regions, and false positives elsewhere.
The values are written with the reference's formats ('%.4f', the score '%f'), so the files read back as the
evaluator reads them.  ``margins_ok`` checks that no overlap lies within ``eps`` of a threshold and that competing
overlaps of one ground truth are either computed from identical boxes or ``eps`` apart; wherever the float64 value
is within 1e-6 of such a decision it is settled with exact rational areas of the reference's (float64) polygon corners.
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

from oracle import kitti_eval as ok

GT_TYPES = ("Car", "Car", "Car", "Pedestrian", "Pedestrian", "Cyclist", "Cyclist", "Van", "Person_sitting", "Truck")
SIZES = {"Car": (1.5, 1.6, 3.9), "Van": (2.2, 1.9, 5.0), "Truck": (3.2, 2.5, 10.0), "Pedestrian": (1.75, 0.6, 0.8),
         "Person_sitting": (1.2, 0.6, 0.8), "Cyclist": (1.7, 0.6, 1.7)}   # h, w, l
DET_OF = {"Car": "Car", "Van": "Car", "Truck": "Car", "Pedestrian": "Pedestrian", "Person_sitting": "Pedestrian",
          "Cyclist": "Cyclist"}
TRUNC = (0.0, 0.0, 0.0, 0.15, 0.16, 0.3, 0.31, 0.5, 0.51, 0.8)
HEIGHTS = (60.0, 90.0, 40.0, 39.99, 40.01, 25.0, 24.99, 30.0, 150.0)
IOU_TARGETS = (0.9, 0.75, 0.71, 0.69, 0.6, 0.51, 0.49, 0.3)


def _fmt_label(t, trunc, occ, alpha, box2d, h, w, l, x, y, z, ry):
    return "%s %.2f %d %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f" % (
        t, trunc, occ, alpha, box2d[0], box2d[1], box2d[2], box2d[3], h, w, l, x, y, z, ry)


def _fmt_det(t, alpha, box2d, h, w, l, x, y, z, ry, score):
    # write_detection_results (train/test_net_det.py:88-123)
    return (t + " -1 -1 " + "%.4f " % alpha + "%.4f %.4f %.4f %.4f " % tuple(box2d) +
            "%.4f %.4f %.4f %.4f %.4f %.4f %.4f %f" % (h, w, l, x, y, z, ry, score))


def _slide(r):
    """Fraction of the length to slide a box along itself for an IoU of r: (1 - f) / (1 + f) = r."""
    return (1.0 - r) / (1.0 + r)


def make_scene(rng, n_obj=8, n_fp=3, dontcare=True, det_rate=1.0, dup_all=False):
    """-> (label lines, result lines) of one image."""
    labels, dets = [], []
    for _ in range(n_obj):
        t = GT_TYPES[rng.integers(len(GT_TYPES))]
        h, w, l = (s * rng.uniform(0.9, 1.1) for s in SIZES[t])
        x, y, z = rng.uniform(-20, 20), rng.uniform(1.0, 2.0), rng.uniform(5, 60)
        ry = rng.uniform(-np.pi, np.pi)
        bh = HEIGHTS[rng.integers(len(HEIGHTS))] if rng.random() < 0.5 else rng.uniform(20, 200)
        bw = rng.uniform(30, 200)
        x1, y1 = rng.uniform(0, 1000), np.round(rng.uniform(100, 200) * 4) / 4   # y1 + 40 is exactly 40 px high
        box = (x1, y1, x1 + bw, y1 + bh)
        trunc = TRUNC[rng.integers(len(TRUNC))]
        occ = int(rng.integers(0, 4))
        alpha = rng.uniform(-np.pi, np.pi)
        labels.append(_fmt_label(t, trunc, occ, alpha, box, h, w, l, x, y, z, ry))
        # the detections start from the values the label file holds ('%.2f'), so a copy is an exact duplicate
        v = [float(f) for f in labels[-1].split()[3:]]
        alpha, box, (h, w, l, x, y, z, ry) = v[0], tuple(v[1:5]), v[5:12]
        bw = box[2] - box[0]
        if dup_all:
            dets.append(_fmt_det(DET_OF[t], alpha + rng.normal(0, 0.3), box, h, w, l, x, y, z, ry,
                                 rng.uniform(0.05, 1.0)))
        if rng.random() > det_rate:
            continue
        dt = DET_OF[t] if rng.random() < 0.9 else ("Car", "Pedestrian", "Cyclist")[rng.integers(3)]
        # the object's detections: duplicate, slid / turned copies, a second detection of one of them
        for k in range(int(rng.integers(1, 4))):
            kind = rng.integers(4)
            if kind == 0:
                f2 = f3 = 0.0
                dry = 0.0
            else:
                f2 = _slide(IOU_TARGETS[rng.integers(len(IOU_TARGETS))]) * rng.choice([-1.0, 1.0])
                f3 = _slide(IOU_TARGETS[rng.integers(len(IOU_TARGETS))]) * rng.choice([-1.0, 1.0])
                dry = rng.uniform(-0.05, 0.05) if kind == 3 else 0.0
            dx = f2 * bw
            dbox = (box[0] + dx, box[1], box[2] + dx, box[3])
            if rng.random() < 0.15:                       # a detection of another height than the object's box
                dbox = (dbox[0], dbox[1], dbox[2], dbox[1] + HEIGHTS[rng.integers(len(HEIGHTS))])
            c, s = np.cos(ry), np.sin(ry)
            dxx, dzz = f3 * l * c, -f3 * l * s              # along the heading (toPolygon's length axis)
            score = rng.uniform(0.05, 1.0)
            dalpha = alpha + rng.normal(0, 0.3)
            row = (dt, dalpha, dbox, h, w, l, x + dxx, y, z + dzz, ry + dry, score)
            dets.append(_fmt_det(*row))
            if rng.random() < 0.15:
                dets.append(_fmt_det(*row[:-1], rng.uniform(0.05, 1.0)))
    if dontcare:
        for _ in range(int(rng.integers(0, 3))):
            x1, y1 = rng.uniform(0, 1100), rng.uniform(100, 250)
            bw, bh = rng.uniform(40, 150), rng.uniform(20, 80)
            labels.append("DontCare -1 -1 -10 %.2f %.2f %.2f %.2f -1 -1 -1 -1000 -1000 -1000 -10"
                          % (x1, y1, x1 + bw, y1 + bh))
            if rng.random() < 0.7:                          # a detection inside it (criterion 0 = 1)
                fx, fy = rng.uniform(0, 0.3), rng.uniform(0, 0.3)
                dbox = (x1 + fx * bw, y1 + fy * bh, x1 + bw * 0.95, y1 + bh * 0.95)
                dets.append(_fmt_det(("Car", "Pedestrian", "Cyclist")[rng.integers(3)], rng.uniform(-3, 3), dbox,
                                     1.5, 1.6, 3.9, rng.uniform(-20, 20), 1.5, rng.uniform(5, 60),
                                     rng.uniform(-3, 3), rng.uniform(0.05, 1.0)))
    for _ in range(int(rng.integers(0, n_fp + 1))):
        x1, y1 = rng.uniform(0, 1100), rng.uniform(100, 250)
        dets.append(_fmt_det(("Car", "Pedestrian", "Cyclist")[rng.integers(3)], rng.uniform(-3, 3),
                             (x1, y1, x1 + rng.uniform(20, 150), y1 + rng.uniform(10, 120)),
                             1.5, 1.6, 3.9, rng.uniform(-20, 20), 1.5, rng.uniform(5, 60), rng.uniform(-3, 3),
                             rng.uniform(0.05, 1.0)))
    return labels, dets


def parse_label_lines(lines):
    from frustum_convnet_b200.kitti_eval import type_code
    rows = [[type_code(t[0]), float(t[1]), int(t[2])] + [float(v) for v in t[3:15]]
            for t in (ln.split() for ln in lines)]
    return np.asarray(rows, dtype=np.float64).reshape(-1, 15)


def parse_result_lines(lines):
    from frustum_convnet_b200.kitti_eval import type_code
    rows = [[type_code(t[0])] + [float(v) for v in t[3:16]] for t in (ln.split() for ln in lines)]
    return np.asarray(rows, dtype=np.float64).reshape(-1, 14)


# ------------------------------------------------------------------------------------------------ exact overlaps
def _area2(p):
    n = len(p)
    return sum(p[i][0] * p[(i + 1) % n][1] - p[(i + 1) % n][0] * p[i][1] for i in range(n))


def _clip(subj, clip):
    """Sutherland-Hodgman in exact arithmetic (correct for convex input, degeneracies included)."""
    sgn = 1 if _area2(clip) >= 0 else -1
    out = list(subj)
    for i in range(len(clip)):
        if not out:
            break
        a, b = clip[i], clip[(i + 1) % len(clip)]
        ex, ey = b[0] - a[0], b[1] - a[1]
        inp, out = out, []
        side = [sgn * (ex * (p[1] - a[1]) - ey * (p[0] - a[0])) for p in inp]
        for j in range(len(inp)):
            k = (j + 1) % len(inp)
            p, q, sp, sq = inp[j], inp[k], side[j], side[k]
            if sp >= 0:
                out.append(p)
            if (sp >= 0) != (sq >= 0):
                t = sp / (sp - sq)
                out.append((p[0] + t * (q[0] - p[0]), p[1] + t * (q[1] - p[1])))
    return out


def exact_overlap(m, d, g):
    """Overlap of metric m (0 image, 1 ground, 2 3-D) as a Fraction: the box values and the float64 polygon corners
    the reference computes (toPolygon) taken as exact, everything after that without rounding.  None when the
    reference divides by zero."""
    F = lambda v: Fraction(float(v))
    crit0 = int(g[ok.G_CODE]) == ok.DONTCARE
    if m == 0:
        x1, y1 = max(F(d[ok.D_X1]), F(g[ok.G_X1])), max(F(d[ok.D_Y1]), F(g[ok.G_Y1]))
        x2, y2 = min(F(d[ok.D_X2]), F(g[ok.G_X2])), min(F(d[ok.D_Y2]), F(g[ok.G_Y2]))
        if x2 - x1 <= 0 or y2 - y1 <= 0:
            return Fraction(0)
        inter = (x2 - x1) * (y2 - y1)
        a = (F(d[ok.D_X2]) - F(d[ok.D_X1])) * (F(d[ok.D_Y2]) - F(d[ok.D_Y1]))
        b = (F(g[ok.G_X2]) - F(g[ok.G_X1])) * (F(g[ok.G_Y2]) - F(g[ok.G_Y1]))
        den = a if crit0 else a + b - inter
        return inter / den if den != 0 else None
    P = lambda poly: [(F(px), F(py)) for px, py in poly]
    gp = P(ok.polygon(g[ok.G_RY], g[ok.G_L], g[ok.G_W], g[ok.G_T1], g[ok.G_T3]))
    dp = P(ok.polygon(d[ok.D_RY], d[ok.D_L], d[ok.D_W], d[ok.D_T1], d[ok.D_T3]))
    inter_poly = _clip(gp, dp)
    inter = abs(_area2(inter_poly)) / 2 if len(inter_poly) >= 3 else Fraction(0)
    ga, da = -_area2(gp) / 2, -_area2(dp) / 2
    if m == 1:
        den = da if crit0 else ga + da - inter
        return inter / den if den != 0 else None
    ymax = min(F(d[ok.D_T2]), F(g[ok.G_T2]))
    ymin = max(F(d[ok.D_T2]) - F(d[ok.D_H]), F(g[ok.G_T2]) - F(g[ok.G_H]))
    inter_vol = inter * max(Fraction(0), ymax - ymin)
    dv = F(d[ok.D_H]) * F(d[ok.D_L]) * F(d[ok.D_W])
    gv = F(g[ok.G_H]) * F(g[ok.G_L]) * F(g[ok.G_W])
    den = dv if crit0 else dv + gv - inter_vol
    return inter_vol / den if den != 0 else None


_GEOMETRY = (ok.D_X1, ok.D_Y1, ok.D_X2, ok.D_Y2, ok.D_H, ok.D_W, ok.D_L, ok.D_T1, ok.D_T2, ok.D_T3, ok.D_RY)


def margins_ok(gt, det, eps=1e-9, band=1e-6):
    """No overlap within eps of 0.5 or 0.7, and the overlaps above 0.5 of one ground truth per metric either come from
    detections with identical geometry or lie eps apart.  The float64 overlaps (error ~1e-15) decide outside a band of
    1e-6 around each decision; inside it the exact overlap (exact_overlap) does."""
    ov = ok.image_pair_overlaps(gt, det)
    exact = {}

    def ex(m, j, k):
        if (m, j, k) not in exact:
            exact[(m, j, k)] = exact_overlap(m, det[j], gt[k])
        return exact[(m, j, k)]

    for m, j, k in zip(*np.nonzero(np.isnan(ov) | (np.abs(ov - 0.5) < band) | (np.abs(ov - 0.7) < band))):
        e = ex(m, j, k)
        if e is None or min(abs(e - Fraction(1, 2)), abs(e - Fraction(7, 10))) < eps:
            return False
    for m in range(3):
        for k in range(ov.shape[2]):
            cand = [j for j in range(ov.shape[1]) if ov[m, j, k] > 0.5 - band]
            for a in range(len(cand)):
                for b in range(a + 1, len(cand)):
                    i, j = cand[a], cand[b]
                    if abs(ov[m, i, k] - ov[m, j, k]) >= band:
                        continue
                    if all(det[i, c] == det[j, c] for c in _GEOMETRY):
                        continue
                    ei, ej = ex(m, i, k), ex(m, j, k)
                    if ei is None or ej is None or abs(ei - ej) < eps:
                        return False
    return True


def make_set(seed, n_images, check_margins=False, **kw):
    """-> (label line lists, result line lists) of n_images images; with check_margins an image is drawn again
    until margins_ok holds."""
    rng = np.random.default_rng(seed)
    labels, results = [], []
    for _ in range(n_images):
        while True:
            lab, det = make_scene(rng, **kw)
            if not check_margins or margins_ok(parse_label_lines(lab), parse_result_lines(det)):
                break
        labels.append(lab)
        results.append(det)
    return labels, results
