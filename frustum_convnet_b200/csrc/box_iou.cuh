// Pairwise rotated-box IoU of the train-branch metrics (SURVEY.md 8(f)-1): replaces the CPU Boost.Geometry
// call `rbbox_iou_3d_pair` (ops/pybind11/box_ops.h:173-260, called at models/det_base.py:495) that forces a
// device->host copy of every predicted box per training step.
//
// The arithmetic lives in this header as plain C++ so that the CPU tests can compile the same source for the host
// (g++) and check it without a GPU: tests/test_box_iou_cpu.py against oracle/box_iou.py, and
// tests/test_box_iou_exact_cpu.py against exact rational arithmetic with and without multiply-add contraction
// (nvcc contracts; the five kernels that inline rbbox_iou_pair are pinned on the device by
// tests/test_gpu_box_iou_exact.py).  The kernels in box_iou.cu only add the thread mapping.  No part of the
// product calls the host build.
#pragma once

#ifdef __CUDACC__
#define FCN_HD __host__ __device__ __forceinline__
#else
#define FCN_HD inline
#endif

namespace fcn {

// The polygon clip is written once for the scalar type: float for the train metric and NMS (below), double for
// the KITTI evaluator's bird's-eye-view and 3-D overlaps (kitti_eval.cu), which works in float64 like the reference.
template <typename T>
struct Vec2 {
    T x, y;
};
using Pt2 = Vec2<float>;
using Pt2d = Vec2<double>;

// signed area, counter-clockwise positive
template <typename T>
FCN_HD T shoelace_ccw(const Vec2<T> *p, int n) {
    T a = T(0);
    for (int i = 0; i < n; ++i) {
        const Vec2<T> u = p[i], v = p[i + 1 == n ? 0 : i + 1];
        a += u.x * v.y - v.x * u.y;
    }
    return T(0.5) * a;
}

// Sutherland-Hodgman: clip the convex quadrilateral `subj` against the convex quadrilateral `clip` (either
// orientation) and return the signed area (counter-clockwise positive) of the intersection; `*count` receives its
// vertex count.  The last clip edge feeds its vertices straight into the shoelace sum (same terms, same order as
// shoelace_ccw on the stored polygon), so that polygon is never stored.
//
// Each vertex is classified ONCE per clip edge: its side value is computed when it first appears as the next
// vertex `q`, carried into the following iteration as `sp`, and the first vertex's value is kept for the wrap-around.
// Computing it twice (as `sq` of edge j and as `sp` of edge j+1) lets a compiler that contracts multiply-adds
// round the two expressions differently; for a vertex within rounding of the clip line (shared or collinear
// edges: boxes slid along their heading, nested boxes) the two signs then disagree, the clip emits a crossing on
// one edge and drops the vertex on the next, and a triangle of the intersection is lost (IoU errors up to ~0.5).
//
// Vertex counts.  In exact arithmetic a convex polygon gains at most one vertex per clip edge (4 -> 5 -> 6 -> 7 ->
// 8).  Rounding can classify vertices within rounding of the line inconsistently with convexity, and then only the
// counting bound holds: with p vertices kept and n - p dropped the output has p + (sign changes) <= p + 2 min(p, n-p)
// <= floor(3n/2) vertices, i.e. at most 6, 9 and 13 after the first three clip edges (and 19 after the last, which
// is not stored).  The two ping-pong buffers are sized for that (9 + 13 entries), so no vertex is ever dropped.
template <typename T>
FCN_HD T clip_quads_area(const Vec2<T> *subj, const Vec2<T> *clip, int *count) {
    Vec2<T> buf[9 + 13];                  // edges 0, 2 write buf + 9 (<= 6, <= 13); edge 1 writes buf (<= 9)
    int n = 4;
    for (int i = 0; i < 4; ++i) buf[i] = subj[i];
    const T sgn = shoelace_ccw(clip, 4) >= T(0) ? T(1) : T(-1);
    T a2 = T(0);                          // twice the signed area, accumulated by the last clip edge
    for (int e = 0; e < 4 && n > 0; ++e) {
        const Vec2<T> a = clip[e], b = clip[(e + 1) & 3];
        const T ex = b.x - a.x, ey = b.y - a.y;
        const Vec2<T> *in = (e & 1) ? buf + 9 : buf;
        Vec2<T> *o = (e & 1) ? buf : buf + 9;
        const bool last = e == 3;
        int m = 0;
        Vec2<T> first = {T(0), T(0)}, prev = {T(0), T(0)};
        auto emit = [&](const Vec2<T> r) {
            if (!last) {
                o[m] = r;
            } else if (m == 0) {
                first = r;
            } else {
                a2 += prev.x * r.y - r.x * prev.y;
            }
            prev = r;
            ++m;
        };
        const Vec2<T> p0 = in[0];
        const T s0 = sgn * (ex * (p0.y - a.y) - ey * (p0.x - a.x));
        Vec2<T> p = p0;
        T sp = s0;
        for (int j = 0; j < n; ++j) {
            const bool wrap = j + 1 == n;
            const Vec2<T> q = wrap ? p0 : in[j + 1];
            const T sq = wrap ? s0 : sgn * (ex * (q.y - a.y) - ey * (q.x - a.x));
            if (sp >= T(0)) emit(p);
            if ((sp >= T(0)) != (sq >= T(0))) {
                const T t = sp / (sp - sq);
                emit(Vec2<T>{p.x + t * (q.x - p.x), p.y + t * (q.y - p.y)});
            }
            p = q;
            sp = sq;
        }
        if (last && m > 0) a2 += prev.x * first.y - first.x * prev.y;
        n = m;
    }
    *count = n;
    return T(0.5) * a2;
}

// c, q: the 8 corners (x, y, z) of one box pair in the reference's corner order (model_util.py:48-72).
// iou[0] = bird's-eye-view IoU, iou[1] = 3-D IoU; (0, 0) when the BEV polygons do not overlap.
FCN_HD void rbbox_iou_pair(const float *c, const float *q, float *iou) {
    const int order[4] = {6, 7, 4, 5};                       // box_ops.h:206-224
    Pt2 P[4], Q[4];
    // coordinates relative to the first polygon vertex: areas are translation invariant and the fp32 cross
    // products then work on box-sized (metres) instead of scene-sized (tens of metres) magnitudes
    const float ox = c[order[0] * 3 + 0], oz = c[order[0] * 3 + 2];
    for (int i = 0; i < 4; ++i) {
        P[i].x = c[order[i] * 3 + 0] - ox;
        P[i].y = c[order[i] * 3 + 2] - oz;
        Q[i].x = q[order[i] * 3 + 0] - ox;
        Q[i].y = q[order[i] * 3 + 2] - oz;
    }
    iou[0] = 0.f;
    iou[1] = 0.f;
    // Degenerate boxes.  The reference hands Boost un-`correct`ed rings (box_ops.h:206-224); a ring whose signed
    // area is not positive in Boost's clockwise convention (a decoded box with exactly one negative footprint
    // size, e.g. from untrained weights) violates the polygon concept and bg::intersection / bg::union_ are
    // unspecified on it.  Decision (pinned in oracle/box_iou.py and tests/test_box_iou_cpu.py): such a pair
    // scores (0, 0) - an invalid box gets no overlap credit - which keeps 0 <= IoU_3D <= IoU_2D <= 1.  Negative
    // HEIGHTS need no special case: `vol = max(0, area*h)` and `max(0, ymax-ymin)` (box_ops.h:242-245) already
    // yield a zero 3-D IoU, exactly as the reference arithmetic does.
    const float area = -shoelace_ccw(P, 4), qarea = -shoelace_ccw(Q, 4);   // clockwise positive (Boost default)
    if (!(area > 0.f) || !(qarea > 0.f)) return;
    int n;
    float inter = clip_quads_area(P, Q, &n);
    if (n < 3) return;
    inter = inter < 0.f ? -inter : inter;
    if (!(inter > 0.f)) return;
    const float uni = area + qarea - inter;
    const float ymax = c[1] < q[1] ? c[1] : q[1];                          // min of the corner-0 heights
    const float ymin = c[13] > q[13] ? c[13] : q[13];                      // max of the corner-4 heights
    const float h = c[1] - c[13], qh = q[1] - q[13];
    const float dy = ymax - ymin;
    const float inter_vol = inter * (dy > 0.f ? dy : 0.f);
    const float vol = area * h > 0.f ? area * h : 0.f, qvol = qarea * qh > 0.f ? qarea * qh : 0.f;
    iou[0] = inter / uni;
    iou[1] = inter_vol / (vol + qvol - inter_vol);
}

#ifdef __CUDACC__
// The 3-D IoU of the reference's Boost kernels in float64 (rbbox_iou_3d_pair<double>, box_ops.h:206-249, element [1];
// the same arithmetic as rbbox_iou_3d, :85-170): the SUN-RGBD evaluator's overlaps (sunrgbd_eval.cu) and the KITTI
// refinement extractor's detection / ground-truth matching (refine_extract.cu).  Rings are the (x, z) of corners 6, 7,
// 4, 5; a ring that is not clockwise-positive scores 0 (the rule of rbbox_iou_pair above and oracle/box_iou.py).
// std::min / std::max semantics are kept (ternaries), as are the reference's separate products.
__device__ inline double rbbox_iou3d_d(const double *__restrict__ c, const double *__restrict__ q) {
    const int order[4] = {6, 7, 4, 5};
    Pt2d P[4], Q[4];
    for (int i = 0; i < 4; ++i) {
        P[i].x = c[order[i] * 3 + 0];
        P[i].y = c[order[i] * 3 + 2];
        Q[i].x = q[order[i] * 3 + 0];
        Q[i].y = q[order[i] * 3 + 2];
    }
    const double area = -shoelace_ccw(P, 4), qarea = -shoelace_ccw(Q, 4);
    if (!(area > 0.0) || !(qarea > 0.0)) return 0.0;
    int n;
    double inter = clip_quads_area(P, Q, &n);
    if (n < 3) return 0.0;
    inter = fabs(inter);
    if (!(inter > 0.0)) return 0.0;
    const double ymax = q[1] < c[1] ? q[1] : c[1];
    const double ymin = c[13] < q[13] ? q[13] : c[13];
    const double h = c[1] - c[13], qh = q[1] - q[13];
    const double dy = ymax - ymin;
    const double inter_vol = __dmul_rn(inter, 0.0 < dy ? dy : 0.0);
    const double av = __dmul_rn(area, h), qv = __dmul_rn(qarea, qh);
    const double vol = 0.0 < av ? av : 0.0, qvol = 0.0 < qv ? qv : 0.0;
    return inter_vol / __dadd_rn(__dadd_rn(vol, qvol), -inter_vol);
}
#endif

}  // namespace fcn
