"""Exact rotated-box IoU of the train metric (oracle/box_iou.py's formulas) in rational arithmetic, and generators
of the box pairs where a floating-point polygon clip goes wrong.

``exact_iou(c, q)`` takes corners ``(N, 8, 3)`` (float32 or float64; both are dyadic, so ``Fraction`` holds them
exactly) and returns the float64 values of the exact (BEV IoU, 3-D IoU, BEV union area) per pair:

  * BEV polygons are the (x, z) coordinates of corners 6, 7, 4, 5; a ring whose clockwise area is not positive
    scores (0, 0) (the degenerate-ring decision of oracle/box_iou.py);
  * the intersection of the two convex quadrilaterals by Sutherland-Hodgman in exact arithmetic, which is correct
    for convex input including every degeneracy (shared and collinear edges, touching, vertices on edges);
  * ``ymax = min(c[0].y, q[0].y)``, ``ymin = max(c[4].y, q[4].y)``, ``inter_vol = inter * max(0, ymax - ymin)``,
    ``vol = max(0, area * h)``; N != K gives zeros.

Generators.  ``FAMILIES[name](scale, seed, n)`` returns two boxes per pair as ``(ctr (n, 3), head (n,), size
(n, 3))`` float64 arrays; ``corners_f32`` turns them into the float32 corners a kernel sees.  ``SCALES`` are KITTI
cars up to 80 m from the origin, pedestrians, and SUN-RGBD objects (up to 8 m, sizes 0.3-4 m).
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

from oracle import box_iou as ob

BEV_ORDER = (6, 7, 4, 5)


# ------------------------------------------------------------------------------------------------ exact reference
def _area2(p):
    """Twice the signed area (counter-clockwise positive) of a polygon of Fractions."""
    n = len(p)
    return sum(p[i][0] * p[(i + 1) % n][1] - p[(i + 1) % n][0] * p[i][1] for i in range(n))


def _clip(subj, clip):
    s = 1 if _area2(clip) >= 0 else -1
    out = list(subj)
    for i in range(len(clip)):
        if not out:
            break
        a, b = clip[i], clip[(i + 1) % len(clip)]
        ex, ey = b[0] - a[0], b[1] - a[1]
        inp, out = out, []
        side = [s * (ex * (p[1] - a[1]) - ey * (p[0] - a[0])) for p in inp]
        for j in range(len(inp)):
            k = (j + 1) % len(inp)
            p, q, sp, sq = inp[j], inp[k], side[j], side[k]
            if sp >= 0:
                out.append(p)
            if (sp >= 0) != (sq >= 0):
                t = sp / (sp - sq)
                out.append((p[0] + t * (q[0] - p[0]), p[1] + t * (q[1] - p[1])))
    return out


def exact_pair(c, q):
    """One pair of (8, 3) corner arrays -> (iou_bev, iou_3d, union_bev) as floats, computed exactly."""
    P = [(Fraction(float(c[i, 0])), Fraction(float(c[i, 2]))) for i in BEV_ORDER]
    Q = [(Fraction(float(q[i, 0])), Fraction(float(q[i, 2]))) for i in BEV_ORDER]
    area, qarea = -_area2(P) / 2, -_area2(Q) / 2                 # clockwise positive
    if area <= 0 or qarea <= 0:
        return 0.0, 0.0, 0.0
    inter = abs(_area2(_clip(P, Q))) / 2
    union = area + qarea - inter
    if inter == 0:
        return 0.0, 0.0, float(union)
    y = lambda a, i: Fraction(float(a[i, 1]))
    ymax, ymin = min(y(c, 0), y(q, 0)), max(y(c, 4), y(q, 4))
    h, qh = y(c, 0) - y(c, 4), y(q, 0) - y(q, 4)
    inter_vol = inter * max(Fraction(0), ymax - ymin)
    vol, qvol = max(Fraction(0), area * h), max(Fraction(0), qarea * qh)
    return float(inter / union), float(inter_vol / (vol + qvol - inter_vol)), float(union)


def exact_iou(c, q):
    """(N, 8, 3), (K, 8, 3) -> (N, 3) float64: exact BEV IoU, 3-D IoU and BEV union area."""
    c, q = np.asarray(c), np.asarray(q)
    out = np.zeros((c.shape[0], 3))
    if c.shape[0] == 0 or c.shape[0] != q.shape[0]:
        return out
    for n in range(c.shape[0]):
        out[n] = exact_pair(c[n], q[n])
    return out


# ------------------------------------------------------------------------------------------------ rounding bound
U = 2.0 ** -24


def kernel_scale(c, q):
    """Per pair: D = the largest |coordinate| of both BEV polygons after the kernel's float32 shift to the first
    vertex of ``c``, and the sum of the two BEV perimeters."""
    c = np.asarray(c, np.float32)
    q = np.asarray(q, np.float32)
    o = c[:, BEV_ORDER[0]][:, [0, 2]]
    P = (c[:, list(BEV_ORDER)][:, :, [0, 2]] - o[:, None]).astype(np.float64)       # float32 subtraction
    Q = (q[:, list(BEV_ORDER)][:, :, [0, 2]] - o[:, None]).astype(np.float64)
    D = np.maximum(np.abs(P).max((1, 2)), np.abs(Q).max((1, 2)))
    per = lambda X: np.linalg.norm(X - np.roll(X, -1, 1), axis=-1).sum(-1)
    return D, per(P) + per(Q)


K_BOUND = 64


def iou_bound(c, q, union):
    """Per pair: K u D (perim_P + perim_Q) / union, the bound on a float32 IoU that tests/test_box_iou_exact_cpu.py
    derives; 0 where the exact union is 0 (a degenerate ring: the exact result is 0 and so must the kernel's be)."""
    D, per = kernel_scale(c, q)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(union > 0, K_BOUND * U * D * per / union, 0.0)


# ------------------------------------------------------------------------------------------------ generators
SCALES = {
    # centre spread (x, z) around (0, z0), size low / high (l, w, h)
    "kitti": dict(spread=(40.0, 40.0), z0=40.0, lo=(3.0, 1.4, 1.3), hi=(4.5, 1.9, 1.8)),
    "pedestrian": dict(spread=(20.0, 20.0), z0=20.0, lo=(0.5, 0.4, 1.5), hi=(1.0, 0.8, 1.9)),
    "sunrgbd": dict(spread=(4.0, 4.0), z0=4.0, lo=(0.3, 0.3, 0.3), hi=(4.0, 4.0, 2.5)),
}


def _base(scale, rng, n):
    s = SCALES[scale]
    ctr = np.stack([rng.uniform(-s["spread"][0], s["spread"][0], n), rng.uniform(-1.0, 2.0, n),
                    s["z0"] + rng.uniform(-s["spread"][1], s["spread"][1], n)], 1)
    head = rng.uniform(-np.pi, np.pi, n)
    size = rng.uniform(s["lo"], s["hi"], (n, 3))
    return ctr, head, size


def _along(head):
    """Unit vectors of the length (local x) and width (local z) directions in the (x, y, z) frame."""
    L = np.stack([np.cos(head), np.zeros_like(head), -np.sin(head)], 1)
    W = np.stack([np.sin(head), np.zeros_like(head), np.cos(head)], 1)
    return L, W


def _rng(seed, name):
    return np.random.default_rng([seed, sum(map(ord, name))])


def fam_slide_length(scale, seed, n):
    rng = _rng(seed, "slide_length")
    c, h, s = _base(scale, rng, n)
    L, _ = _along(h)
    fr = rng.uniform(-1.1, 1.1, n)
    return (c, h, s), (c + L * (fr * s[:, 0])[:, None], h, s)


def fam_slide_width(scale, seed, n):
    rng = _rng(seed, "slide_width")
    c, h, s = _base(scale, rng, n)
    _, W = _along(h)
    fr = rng.uniform(-1.1, 1.1, n)
    return (c, h, s), (c + W * (fr * s[:, 1])[:, None], h, s)


def fam_heading_delta(scale, seed, n):
    """Slid along the length with a heading that differs by 1e-7 .. 1e-3 rad."""
    rng = _rng(seed, "heading_delta")
    c, h, s = _base(scale, rng, n)
    L, _ = _along(h)
    fr = rng.uniform(-0.9, 0.9, n)
    dh = rng.choice([-1.0, 1.0], n) * 10.0 ** rng.uniform(-7, -3, n)
    return (c, h, s), (c + L * (fr * s[:, 0])[:, None], h + dh, s)


def fam_tiny_rotation(scale, seed, n):
    """Nearly identical boxes a tiny rotation apart: the intersection is an octagon (the most vertices a clip of
    two convex quadrilaterals has)."""
    rng = _rng(seed, "tiny_rotation")
    c, h, s = _base(scale, rng, n)
    dh = rng.choice([-1.0, 1.0], n) * 10.0 ** rng.uniform(-4, -2, n)
    return (c, h, s), (c, h + dh, s)


def fam_nested_shared_edge(scale, seed, n):
    """A shorter box inside, sharing the +l/2 face (one edge), or shorter and narrower sharing a corner (two)."""
    rng = _rng(seed, "nested_shared_edge")
    c, h, s = _base(scale, rng, n)
    L, W = _along(h)
    fl, fw = rng.uniform(0.1, 0.95, n), np.where(rng.random(n) < 0.5, 1.0, rng.uniform(0.2, 0.95, n))
    sq = s * np.stack([fl, fw, np.ones(n)], 1)
    cq = c + L * ((s[:, 0] - sq[:, 0]) / 2)[:, None] + W * ((s[:, 1] - sq[:, 1]) / 2)[:, None]
    return (c, h, s), (cq, h, sq)


def fam_touching(scale, seed, n):
    """Touching along a long edge (slid along it) or at a corner: exact IoU 0."""
    rng = _rng(seed, "touching")
    c, h, s = _base(scale, rng, n)
    L, W = _along(h)
    corner = rng.random(n) < 0.5
    fr = np.where(corner, 1.0, rng.uniform(-0.9, 0.9, n))
    return (c, h, s), (c + W * s[:, 1:2] + L * (fr * s[:, 0])[:, None], h, s)


def fam_vertex_on_edge(scale, seed, n):
    """The second box turned by 0.2 .. 1.2 rad with one of its corners on an edge of the first."""
    rng = _rng(seed, "vertex_on_edge")
    c, h, s = _base(scale, rng, n)
    L, W = _along(h)
    th = h + rng.uniform(0.2, 1.2, n) * rng.choice([-1.0, 1.0], n)
    sq = rng.uniform(SCALES[scale]["lo"], SCALES[scale]["hi"], (n, 3))
    Lq, Wq = _along(th)
    on_edge = c + W * (s[:, 1] / 2)[:, None] + L * (rng.uniform(-0.4, 0.4, n) * s[:, 0])[:, None]
    # corner (-l/2, -w/2) of the second box on the +w/2 edge of the first; the box extends outwards
    cq = on_edge + Lq * (sq[:, 0] / 2)[:, None] + Wq * (sq[:, 1] / 2)[:, None]
    return (c, h, s), (cq, th, sq)


def fam_containment(scale, seed, n):
    """A smaller box strictly inside (any heading), or the same box (identical)."""
    rng = _rng(seed, "containment")
    c, h, s = _base(scale, rng, n)
    L, W = _along(h)
    same = rng.random(n) < 0.25
    r = np.minimum(s[:, 0], s[:, 1]) * rng.uniform(0.1, 0.35, n)        # half-diagonal of the inner footprint
    sq = np.stack([r * np.sqrt(2.0), r * np.sqrt(2.0), s[:, 2]], 1)
    off = (L * (rng.uniform(-1, 1, n) * (s[:, 0] / 2 - r))[:, None]
           + W * (rng.uniform(-1, 1, n) * (s[:, 1] / 2 - r))[:, None])
    cq = np.where(same[:, None], c, c + off)
    hq = np.where(same, h, rng.uniform(-np.pi, np.pi, n))
    return (c, h, s), (cq, hq, np.where(same[:, None], s, sq))


def fam_axis_headings(scale, seed, n):
    """Headings 0, +-pi/2, +-pi and each of them +-1 float32 ulp, slid along the length or the width."""
    rng = _rng(seed, "axis_headings")
    c, _, s = _base(scale, rng, n)
    ax = np.float32(rng.choice([0.0, np.pi / 2, -np.pi / 2, np.pi, -np.pi], n))
    def ulp(a, k):
        return np.where(k > 0, np.nextafter(a, np.float32(np.inf)),
                        np.where(k < 0, np.nextafter(a, np.float32(-np.inf)), a))
    h = ulp(ax, rng.integers(-1, 2, n)).astype(np.float64)
    hq = ulp(ax, rng.integers(-1, 2, n)).astype(np.float64)
    L, W = _along(h)
    d = np.where((rng.random(n) < 0.5)[:, None], L * (rng.uniform(-0.9, 0.9, n) * s[:, 0])[:, None],
                 W * (rng.uniform(-0.9, 0.9, n) * s[:, 1])[:, None])
    return (c, h, s), (c + d, hq, s)


def fam_quarter_turn(scale, seed, n):
    """Square footprints a quarter turn apart, slid along one side."""
    rng = _rng(seed, "quarter_turn")
    c, h, s = _base(scale, rng, n)
    s[:, 1] = s[:, 0]
    L, _ = _along(h)
    return (c, h, s), (c + L * (rng.uniform(-0.9, 0.9, n) * s[:, 0])[:, None], h + np.pi / 2, s)


def fam_heights(scale, seed, n):
    """Overlapping footprints with equal, touching (ymax == ymin), disjoint and negative heights.  Centres and heights
    on a 2^-6 grid so that the corner heights are exact in float32."""
    rng = _rng(seed, "heights")
    c, h, s = _base(scale, rng, n)
    L, _ = _along(h)
    q = lambda x: np.round(x * 64) / 64
    c[:, 1], s[:, 2] = q(c[:, 1]), np.maximum(q(s[:, 2]), 0.25)
    kind = rng.integers(0, 4, n)
    hq = s[:, 2].copy()
    cy = c[:, 1].copy()
    cy = np.where(kind == 1, c[:, 1] + (s[:, 2] + hq) / 2, cy)                  # touching
    cy = np.where(kind == 2, c[:, 1] + s[:, 2] + q(rng.uniform(0.1, 1.0, n)), cy)   # disjoint
    hq = np.where(kind == 3, -hq, hq)                                              # negative height
    cq = c + L * (rng.uniform(-0.6, 0.6, n) * s[:, 0])[:, None]
    cq[:, 1] = cy
    return (c, h, s), (cq, h, np.stack([s[:, 0], s[:, 1], hq], 1))


def fam_negative_sizes(scale, seed, n):
    """One negative footprint size (an invalid counter-clockwise ring: (0, 0)) or two (the box turned by pi)."""
    rng = _rng(seed, "negative_sizes")
    c, h, s = _base(scale, rng, n)
    L, _ = _along(h)
    kind = rng.integers(0, 3, n)
    sign = np.ones((n, 3))
    sign[kind == 0, 0] = -1
    sign[kind == 1, 1] = -1
    sign[kind == 2, :2] = -1
    return (c, h, s), (c + L * (rng.uniform(-0.5, 0.5, n) * s[:, 0])[:, None], h, s * sign)


FAMILIES = {
    "slide_length": fam_slide_length,
    "slide_width": fam_slide_width,
    "heading_delta": fam_heading_delta,
    "tiny_rotation": fam_tiny_rotation,
    "nested_shared_edge": fam_nested_shared_edge,
    "touching": fam_touching,
    "vertex_on_edge": fam_vertex_on_edge,
    "containment": fam_containment,
    "axis_headings": fam_axis_headings,
    "quarter_turn": fam_quarter_turn,
    "heights": fam_heights,
    "negative_sizes": fam_negative_sizes,
}


def corners_f32(box):
    ctr, head, size = box
    return ob.box3d_corners(ctr, head, size).astype(np.float32)


def family_corners(name, scale, seed, n):
    """Float32 corners (A, B) of one family at one scale."""
    a, b = FAMILIES[name](scale, seed, n)
    return corners_f32(a), corners_f32(b)
