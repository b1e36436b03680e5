"""Rotated-box IoU pinned against exact rational arithmetic (tests/iou_exact_ref.py) on the CPU: the float64 oracles
(oracle/box_iou.py and the pair IoU of oracle/nms.py) and csrc/box_iou.cuh compiled with g++ both without and with
multiply-add contraction, on the pair families where a floating-point polygon clip goes wrong (collinear and shared
edges, touching boxes, vertices on edges, tiny rotations, axis headings +-1 ulp, degenerate heights and sizes) at
KITTI-car, pedestrian and SUN-RGBD scales, in both argument orders.

Bound of the float32 header.  With u = 2^-24, D the largest |coordinate| of the two BEV polygons after the
kernel's shift to the first vertex of its first argument, and perim_P + perim_Q the two perimeters:

    |IoU - IoU_exact| <= K u D (perim_P + perim_Q) / union,   K = 64, for the BEV and the 3-D IoU
    (``iou_bound`` of tests/iou_exact_ref.py).

  * The shift is one correctly rounded subtraction per coordinate, so every shifted coordinate is within u D of
    the exact value: the errors scale with the local extent, not with the distance from the origin.
  * A side value ex*(py - ay) - ey*(px - ax) is computed within ~4 u D^2 (two products of differences, one
    difference, a possible contraction).  With consistent classification a vertex that the sign puts on the wrong
    side of a clip line lies within ~4 u D of it, so keeping or dropping it moves the polygon boundary by that
    much along the adjacent edges; a crossing point t = sp / (sp - sq) has a few u relative error in t, i.e. lies
    within a few u D of both lines it joins, even when its position ALONG the line is ill-conditioned (nearly
    parallel edges).  Each boundary point of the computed intersection is therefore within ~8 u D of the exact
    boundary, and the intersection area is within ~8 u D perim_I <= 8 u D (perim_P + perim_Q) of the exact one.
  * The shoelace sums of the intersection (<= 8 vertices in exact arithmetic) and of the two quadrilaterals
    round each product of coordinates (<= D^2) and each partial sum: <= ~(2 * 8 + 2 * 4) u D^2 in total, and
    D <= (perim_P + perim_Q) / 2 for overlapping polygons.  The union's error is the sum of those of the areas.
  * IoU = I / U: |dIoU| <= (|dI| + IoU |dU|) / U <= 2 (|dI| + |dA| + |dB|) / U.  These add up to ~44; K = 64
    leaves room for the final divisions.  The 3-D IoU divides I dy by vol + qvol - I dy >= U dy (both heights
    are >= dy), so the same bound holds; the heights themselves are compared and subtracted exactly or within u.

The measured worst fraction of the bound is printed per build (pytest -s).  A clip that classifies a vertex
twice with differently contracted expressions exceeds it by four orders of magnitude on the slide and shared-edge
families (errors up to ~0.5): without contraction both expressions round the same way and the defect hides.
"""
import ctypes
import os

import numpy as np
import pytest

import iou_exact_ref as ex
from oracle import box_iou as ob
from oracle import nms as onms
from toolchain import fma_cpu, host_library

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, "frustum_convnet_b200", "csrc", "box_iou.cuh")
N_PAIRS = 500
SEED = 7
MODES = {"no_contraction": ("-ffp-contract=off",), "contracted": ("-mfma", "-ffp-contract=fast")}

HARNESS = r'''
#include "%s"
extern "C" void host_rbbox_iou(int M, const float* c, const float* q, float* out) {
    for (int n = 0; n < M; ++n) fcn::rbbox_iou_pair(c + 24 * n, q + 24 * n, out + 2 * n);
}
// vertex count of the BEV intersection, in the kernel's shifted frame
extern "C" void host_clip_count(int M, const float* c, const float* q, int* cnt) {
    const int order[4] = {6, 7, 4, 5};
    for (int n = 0; n < M; ++n) {
        const float *a = c + 24 * n, *b = q + 24 * n;
        fcn::Pt2 P[4], Q[4];
        for (int i = 0; i < 4; ++i) {
            P[i].x = a[order[i] * 3] - a[18];  P[i].y = a[order[i] * 3 + 2] - a[20];
            Q[i].x = b[order[i] * 3] - a[18];  Q[i].y = b[order[i] * 3 + 2] - a[20];
        }
        fcn::clip_quads_area(P, Q, cnt + n);
    }
}
'''


@pytest.fixture(scope="module")
def host_lib():
    return {mode: host_library(HARNESS % HDR, flags) for mode, flags in MODES.items()
            if mode != "contracted" or fma_cpu()}


def _run(lib, c, q):
    c = np.ascontiguousarray(c, dtype=np.float32)
    q = np.ascontiguousarray(q, dtype=np.float32)
    out = np.full((c.shape[0], 2), np.nan, dtype=np.float32)
    P = ctypes.c_void_p
    lib.host_rbbox_iou(ctypes.c_int(c.shape[0]), P(c.ctypes.data), P(q.ctypes.data), P(out.ctypes.data))
    return out.astype(np.float64)


def _counts(lib, c, q):
    c = np.ascontiguousarray(c, dtype=np.float32)
    q = np.ascontiguousarray(q, dtype=np.float32)
    cnt = np.zeros(c.shape[0], dtype=np.int32)
    P = ctypes.c_void_p
    lib.host_clip_count(ctypes.c_int(c.shape[0]), P(c.ctypes.data), P(q.ctypes.data), P(cnt.ctypes.data))
    return cnt


_CACHE = {}


def family(name, scale):
    """Float32 corners (A, B) and the exact (iou_bev, iou_3d, union) of one family, computed once per session."""
    key = (name, scale)
    if key not in _CACHE:
        A, B = ex.family_corners(name, scale, SEED, N_PAIRS)
        _CACHE[key] = (A, B, ex.exact_iou(A, B))
    return _CACHE[key]


def check_within_bound(got, c, q, want, what):
    """got (N, 2) against the exact (N, 3); returns the worst fraction of the bound."""
    b = ex.iou_bound(c, q, want[:, 2])
    assert np.isfinite(got).all(), what
    assert (got >= 0).all() and (got <= 1 + 1e-6).all(), what
    err = np.abs(got - want[:, :2])
    bad = err > b[:, None]
    if bad.any():
        i = int(np.nonzero(bad.any(1))[0][0])
        raise AssertionError("%s: %d of %d pairs out of bound; first pair %d: got %s exact %s bound %.3g" % (
            what, int(bad.any(1).sum()), len(got), i, got[i], want[i, :2], b[i]))
    with np.errstate(divide="ignore", invalid="ignore"):
        frac = np.where(b[:, None] > 0, err / b[:, None], 0.0)
    return float(frac.max())


# ================================================================================ the exact reference itself
def _boxes(ctr, head, size):
    return ob.box3d_corners(np.asarray(ctr, float), np.asarray(head, float), np.asarray(size, float)).astype(np.float32)


def test_exact_reference_closed_forms():
    size = [[4.0, 2.0, 1.5]]
    base = _boxes([[1.0, 1.0, 10.0]], [0.0], size)
    iou = lambda q: ex.exact_iou(base, q)[0, :2]
    assert iou(base).tolist() == [1.0, 1.0]
    assert iou(_boxes([[2.0, 1.0, 10.0]], [0.0], size)).tolist() == [0.6, 0.6]              # 6 / (16 - 6)
    assert iou(_boxes([[2.0, 1.5, 10.0]], [0.0], size)).tolist() == [0.6, 6.0 / 18.0]       # heights overlap 1.0
    assert iou(_boxes([[1.0, 1.0, 10.0]], [np.pi / 2], size)).tolist() == [1 / 3, 1 / 3]    # 4 / (16 - 4)
    assert iou(_boxes([[9.0, 1.0, 10.0]], [0.0], size)).tolist() == [0.0, 0.0]
    assert iou(_boxes([[5.0, 1.0, 10.0]], [0.0], size)).tolist() == [0.0, 0.0]              # touching edge
    assert iou(_boxes([[1.0, 4.0, 10.0]], [0.0], size)).tolist() == [1.0, 0.0]              # no height overlap
    sq = [[2.0, 2.0, 1.0]]
    a = _boxes([[0.0, 0.0, 5.0]], [0.0], sq)
    b = _boxes([[0.0, 0.0, 5.0]], [np.pi / 4], sq)
    oct_area = 8.0 * (np.sqrt(2.0) - 1.0)
    assert ex.exact_iou(a, b)[0, 0] == pytest.approx(oct_area / (8.0 - oct_area), abs=1e-6)   # float32 corners
    # degenerate ring (one negative footprint size) scores (0, 0); N != K and N == 0 give zeros
    assert not ex.exact_iou(base, _boxes([[1.0, 1.0, 10.0]], [0.0], [[-4.0, 2.0, 1.5]]))[:, :2].any()
    assert ex.exact_iou(base, np.zeros((0, 8, 3))).shape == (1, 3)
    assert not ex.exact_iou(np.concatenate([base, base]), base).any()


def test_oracle_matches_exact_on_fixture():
    g = dict(np.load(os.path.join(ROOT, "tests", "golden", "box_pairs.npz")))
    want = ex.exact_iou(g["pr_corners"], g["gt_corners"])
    got = ob.rbbox_iou_3d_pair(g["pr_corners"], g["gt_corners"])
    assert np.abs(got - want[:, :2]).max() <= 1e-9
    assert 0 < want[:, 1].mean() < want[:, 0].mean() < 1


@pytest.mark.parametrize("scale", list(ex.SCALES))
def test_oracles_match_exact_on_every_family(scale):
    """oracle/box_iou.py, and the pair IoU oracle/nms.py computes from its own float64 corners, within 1e-9 of
    exact arithmetic: the oracles remain a trustworthy proxy for the keep lists of the NMS and detect tests."""
    worst = 0.0
    for name in ex.FAMILIES:
        A, B, want = family(name, scale)
        for c, q in ((A, B), (B, A)):
            got = ob.rbbox_iou_3d_pair(c, q)
            worst = max(worst, float(np.abs(got - want[:, :2]).max()))
        # the NMS path: dets (cx, cy, cz, l, w, h, ry) -> float64 corners -> the same pair IoU
        a, b = ex.FAMILIES[name](scale, SEED, N_PAIRS)
        dets = lambda box: np.concatenate([box[0], box[2], box[1][:, None]], 1).astype(np.float32)
        ca, cb = onms.boxes3d2corners(dets(a)), onms.boxes3d2corners(dets(b))
        exact64 = ex.exact_iou(ca[:40], cb[:40])[:, 1]
        nms_iou = np.array([ob.rbbox_iou_3d_pair(ca[i:i + 1], cb[i:i + 1])[0, 1] for i in range(40)])
        worst = max(worst, float(np.abs(nms_iou - exact64).max()))
    assert worst <= 1e-9, worst


@pytest.mark.parametrize("mode", list(MODES))
def test_header_within_bound_of_exact_in_both_contraction_modes(host_lib, mode):
    if mode not in host_lib:
        pytest.skip("the host CPU has no FMA instructions")
    lib = host_lib[mode]
    worst, rows = 0.0, []
    for scale in ex.SCALES:
        for name in ex.FAMILIES:
            A, B, want = family(name, scale)
            for tag, (c, q) in (("", (A, B)), (" swapped", (B, A))):
                f = check_within_bound(_run(lib, c, q), c, q, want, "%s %s/%s%s" % (mode, scale, name, tag))
                worst = max(worst, f)
                rows.append((scale, name + tag, f))
    print("\n%s: worst fraction of the bound %.3g" % (mode, worst))
    for scale, name, f in sorted(rows, key=lambda r: -r[2])[:5]:
        print("  %-10s %-28s %.3g" % (scale, name, f))
    # exact zeros stay zeros: no overlap credit for touching boxes beyond rounding, none for invalid rings
    for scale in ex.SCALES:
        A, B, want = family("negative_sizes", scale)
        got = _run(lib, A, B)
        assert not got[want[:, 0] == 0].any()


def test_intersection_reaches_eight_vertices_within_bound(host_lib):
    """Nearly identical rotated rectangles intersect in an octagon, the most vertices the exact clip of two convex
    quadrilaterals has; the tiny-rotation family reaches it on most pairs, in both builds, within the bound."""
    for mode, lib in host_lib.items():
        for scale in ex.SCALES:
            A, B, want = family("tiny_rotation", scale)
            for c, q in ((A, B), (B, A)):
                cnt = _counts(lib, c, q)
                assert (cnt == 8).mean() >= 0.4, (mode, scale, np.bincount(cnt))
                check_within_bound(_run(lib, c, q), c, q, want, "%s %s/tiny_rotation" % (mode, scale))
