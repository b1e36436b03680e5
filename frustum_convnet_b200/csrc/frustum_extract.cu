// KITTI frustum extraction on the device (C ABI section (15)): extract_frustum_data_rgb_detection of
// kitti/prepare_data.py:462-568 for several frames and all their 2-D detections in one pair of calls.
//
// The reference re-masks the whole scan for every detection and projects every scan twice.  Here:
//   fcn_frustum_extract_count  flags    (csrc/frustum_fov.cu, as the scans and compact below) one thread per scan
//                                       point: velo -> rect -> image in float64 (every product and sum rounded
//                                       separately, kitti_util.py:172-210) and the image test of get_lidar_in_image_fov
//                                       (draw_util.py:15-18);
//                              scan     exclusive sum of the flags over all frames (frames stay contiguous, scan order
//                                       is kept): the position of every in-image point;
//                              compact  the in-image points, recomputed, stored at those positions: float32 rect and
//                                       intensity (prepare_data.py:506-508) plus float64 u, v;
//                              count    one CTA per detection over its frame's in-image points only: the clipped box
//                                       (:522-524), the box test (:527-532), the frustum angle (:537-543) and the
//                                       drop rules (:546-548);
//                              scans    exclusive sums over the kept detections and their point counts, then info;
//   fcn_frustum_extract_write  write    one CTA per kept detection: the box test again, a block scan for stable
//                                       positions, the points scattered in scan order, and the per-detection values.
//
// fcn_frame_extract (section (21)) runs the same count and write kernels over fixed capacities with every size read
// on the device, around the frame kernels of csrc/frame_extract.cu: frame_setup and frame_pack before the count
// entry's stages, frame_slots between them and fx_write_kernel over every slot.
#include <cmath>

#include "common.cuh"
#include "frame_extract.cuh"
#include "frustum_fov.cuh"
#include "input_builder.cuh"

namespace fcn {

// np.clip(a, 0, hi): NaN stays NaN
__device__ __forceinline__ double fx_clip(double a, double hi) {
    const double c = a < 0.0 ? 0.0 : a;
    return c > hi ? hi : c;
}

__device__ __forceinline__ bool fx_in_box(double u, double v, const double *b) {
    return u < b[2] && u >= b[0] && v < b[3] && v >= b[1];
}

__global__ void __launch_bounds__(FX_THREADS)
fx_count_kernel(int num_frames, const int32_t *__restrict__ so, const fcn_frustum_frame *__restrict__ frames,
                const double *__restrict__ boxes, const int32_t *__restrict__ det_frame,
                const int32_t *__restrict__ pos, const double *__restrict__ fov_u, const double *__restrict__ fov_v,
                int32_t *__restrict__ det_points, int32_t *__restrict__ keep, long long *__restrict__ cnt,
                double *__restrict__ box_ws, double *__restrict__ angle_ws, int32_t *__restrict__ bad) {
    const int d = blockIdx.x, f = det_frame[d];
    if (f < 0 || f >= num_frames) {
        if (threadIdx.x == 0) {
            job_words(d, true, 0, det_points, keep, cnt);
            atomicAdd(bad, 1);
        }
        return;
    }
    const fcn_frustum_frame *fr = frames + f;
    double b[4];
    b[0] = fx_clip(boxes[4 * d + 0], (double)(fr->width - 1));
    b[1] = fx_clip(boxes[4 * d + 1], (double)(fr->height - 1));
    b[2] = fx_clip(boxes[4 * d + 2], (double)(fr->width - 1));
    b[3] = fx_clip(boxes[4 * d + 3], (double)(fr->height - 1));
    const int p0 = pos[so[f]], p1 = pos[so[f + 1]];
    int c, l;
    job_count<false>(p0, p1, c, l, [&](int i, int &n, int &) { n += fx_in_box(fov_u[i], fov_v[i], b); });
    if (threadIdx.x == 0) {
        job_words(d, b[3] - b[1] < 5.0 || b[2] - b[0] < 1.0 || c < 1, c, det_points, keep, cnt);
        const RectProjection rp(b, fr->P);
        double x, y;
        rp.at(20.0, &x, &y);
        angle_ws[d] = -atan2(20.0, x);
#pragma unroll
        for (int j = 0; j < 4; ++j) box_ws[4 * d + j] = b[j];
    }
}

__global__ void __launch_bounds__(FX_THREADS)
fx_write_kernel(int num_kept, long long num_out, const int32_t *__restrict__ so,
                const fcn_frustum_frame *__restrict__ frames, const int32_t *__restrict__ det_frame,
                const int32_t *__restrict__ det_points, const int32_t *__restrict__ keep_pos,
                const long long *__restrict__ cnt_pos, const double *__restrict__ box_ws,
                const double *__restrict__ angle_ws, const int32_t *__restrict__ pos,
                const float4 *__restrict__ fov_pts, const double *__restrict__ fov_u,
                const double *__restrict__ fov_v, float4 *__restrict__ points, int32_t *__restrict__ offsets,
                double *__restrict__ angle, double *__restrict__ box2d, double *__restrict__ P,
                int32_t *__restrict__ det_index) {
    // kept_slot's guard spelled out: offsets[k + 1] is written with the per-detection values, where this kernel has
    // always written it (kept_slot's earlier store changes its instruction schedule)
    const int d = blockIdx.x, c = det_points[d];
    if (c < 0) return;
    const int k = keep_pos[d];
    const long long base = cnt_pos[d];
    if (k >= num_kept || base + c > num_out) return;
    const int f = det_frame[d];
    const double *b = box_ws + 4 * d;
    if (threadIdx.x < 12) P[12 * k + threadIdx.x] = frames[f].P[threadIdx.x];
    if (threadIdx.x < 4) box2d[4 * k + threadIdx.x] = b[threadIdx.x];
    if (threadIdx.x == 0) {
        offsets[k + 1] = (int32_t)(base + c);
        angle[k] = angle_ws[d];
        det_index[k] = d;
    }
    const double bb[4] = {b[0], b[1], b[2], b[3]};
    job_scatter(pos[so[f]], pos[so[f + 1]], c, base, [&](int i) { return fx_in_box(fov_u[i], fov_v[i], bb); },
                [&](long long o, int i) { points[o] = fov_pts[i]; });
}

// ------------------------------------------------------------------------------------------------ host side
struct FxWs : FovWs {
    double *box, *angle;
};

static cudaError_t fx_layout(const fcn_frustum_extract_args *a, Carve &c, FxWs &w) {
    const cudaError_t e = fov_carve(c, a->num_points, a->num_dets, true, w);
    w.box = (double *)c.take((size_t)a->num_dets * 32);
    w.angle = (double *)c.take((size_t)a->num_dets * 8);
    return e;
}

// Host-side checks shared by every entry: counts, pointers, the scans.  Sets *max_n to the largest scan.
static int fx_check(const fcn_frustum_extract_args *a, const char *fn, int *max_n) {
    if (a == nullptr) return invalid(fn, "NULL args");
    if (a->num_frames < 0 || a->num_points < 0 || a->num_dets < 0)
        return invalid(fn, "negative count (num_frames, num_points, num_dets must be >= 0)");
    if (a->num_frames > 65535 || a->num_points > (1 << 30) || a->num_dets > (1 << 28))
        return invalid(fn, "too large (num_frames <= 65535, num_points <= 2^30, num_dets <= 2^28)");
    *max_n = 0;
    if (a->num_frames == 0 || a->num_dets == 0) return FCN_OK;
    if (!a->scan_offsets || !a->frames || !a->boxes || !a->det_frame || (a->num_points > 0 && !a->scans))
        return invalid(fn, "NULL pointer");
    return check_scans(fn, a->host_scan_offsets, a->num_frames, a->num_points, a->scans, 16, max_n);
}

static int fx_prepare(const fcn_frustum_extract_args *a, const char *fn, FxWs &w, int *max_n) {
    const int st = fx_check(a, fn, max_n);
    if (st != FCN_OK || a->num_frames == 0 || a->num_dets == 0) return st;
    if (!a->workspace || !a->info || !a->det_points) return invalid(fn, "NULL workspace, info or det_points");
    return carve_workspace(fn, "frustum_extract", a->workspace, a->workspace_bytes,
                           [&](Carve &c) { return fx_layout(a, c, w); });
}

struct FrameWs : FxWs {
    float4 *packed;
    int32_t *so, *det_frame, *det_points, *c2, *kpos;
    long long *base, *info;
};

static cudaError_t frame_layout(const fcn_frame_extract_args *a, Carve &c, FrameWs &w) {
    const size_t F = (size_t)a->num_frames, FP = F * a->scan_capacity, FD = F * a->det_capacity;
    const cudaError_t e = fov_carve(c, (int)FP, (int)FD, true, w);
    w.box = (double *)c.take(FD * 32);
    w.angle = (double *)c.take(FD * 8);
    w.packed = (float4 *)c.take(FP * 16);
    w.so = (int32_t *)c.take((F + 1) * 4);
    w.det_frame = (int32_t *)c.take(FD * 4);
    w.det_points = (int32_t *)c.take(FD * 4);
    w.c2 = (int32_t *)c.take(FD * 4);
    w.kpos = (int32_t *)c.take(FD * 4);
    w.base = (long long *)c.take(FD * 8);
    w.info = (long long *)c.take(32);
    return e;
}

// the capacities, which alone size the workspace
static int frame_check_sizes(const fcn_frame_extract_args *a, const char *fn) {
    if (a == nullptr) return invalid(fn, "NULL args");
    const long long F = a->num_frames, P = a->scan_capacity, D = a->det_capacity, Po = a->out_capacity;
    if (F < 1 || P < 1 || D < 1 || Po < 1) return invalid(fn, "capacities must be >= 1");
    if (F > 65535 || F * P > (1 << 30) || F * D > (1 << 28) || Po >= (1 << 24) || F * Po + F * D >= (1LL << 31))
        return invalid(fn, "too large (F <= 65535, F * P <= 2^30, F * D <= 2^28, P_out < 2^24, "
                           "F * (P_out + D) < 2^31)");
    return FCN_OK;
}

static int frame_check(const fcn_frame_extract_args *a, const char *fn) {
    const int st = frame_check_sizes(a, fn);
    if (st != FCN_OK) return st;
    if (!a->scans || !a->scan_counts || !a->frames || !a->boxes || !a->det_class || !a->det_prob || !a->det_counts ||
        !a->status)
        return invalid(fn, "NULL input");
    if (!a->points || !a->offsets || !a->frustum_angle || !a->box2d || !a->P || !a->det_index || !a->valid ||
        !a->cls_index || !a->seg || !a->seg_class || !a->rgb_prob)
        return invalid(fn, "NULL output");
    if (((uintptr_t)a->scans & 15) != 0 || ((uintptr_t)a->points & 15) != 0)
        return invalid(fn, "scans and points must be 16-byte aligned");
    return FCN_OK;
}

}  // namespace fcn

using namespace fcn;

extern "C" long long fcn_frame_extract_workspace_bytes(const fcn_frame_extract_args *a) {
    if (frame_check_sizes(a, __func__) != FCN_OK) return -1;
    FrameWs w;
    return workspace_size(__func__, [&](Carve &c) { return frame_layout(a, c, w); });
}

extern "C" int fcn_frame_extract(const fcn_frame_extract_args *a, fcn_stream_t stream) {
    int st = frame_check(a, __func__);
    if (st != FCN_OK) return st;
    FrameWs w;
    st = carve_workspace(__func__, "frame_extract", a->workspace, a->workspace_bytes,
                         [&](Carve &c) { return frame_layout(a, c, w); });
    if (st != FCN_OK) return st;
    cudaStream_t s = (cudaStream_t)stream;
    const int F = a->num_frames, P = a->scan_capacity, B = F * a->det_capacity;
    FCN_CUDA(frame_setup(*a, w.so, w.det_frame, w.packed, s));
    // flags past the packed points are never written; the exclusive scan of the in-image stage reads them only after
    // every position it is asked for
    FCN_CUDA(fov_stage(w, F * P, B, F, P, w.packed, w.so, a->frames, s));
    fx_count_kernel<<<B, FX_THREADS, 0, s>>>(F, w.so, a->frames, a->boxes, w.det_frame, w.pos, w.fov_u, w.fov_v,
                                             w.det_points, w.keep, w.cnt, w.box, w.angle, w.bad);
    FCN_LAUNCH_CHECK();
    FCN_CUDA(job_totals(w, B, w.info, s));
    FCN_CUDA(frame_slots(*a, w.det_points, w.c2, w.kpos, w.base, s));
    fx_write_kernel<<<B, FX_THREADS, 0, s>>>(B, (long long)F * a->out_capacity, w.so, a->frames, w.det_frame, w.c2,
                                             w.kpos, w.base, w.box, w.angle, w.pos, w.fov_pts, w.fov_u, w.fov_v,
                                             (float4 *)a->points, a->offsets, a->frustum_angle, a->box2d, a->P,
                                             a->det_index);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

extern "C" long long fcn_frustum_extract_workspace_bytes(const fcn_frustum_extract_args *a) {
    int max_n;
    if (fx_check(a, __func__, &max_n) != FCN_OK) return -1;
    if (a->num_frames == 0 || a->num_dets == 0) return 0;
    FxWs w;
    return workspace_size(__func__, [&](Carve &c) { return fx_layout(a, c, w); });
}

extern "C" int fcn_frustum_extract_count(const fcn_frustum_extract_args *a, fcn_stream_t stream) {
    FxWs w;
    int max_n;
    const int st = fx_prepare(a, __func__, w, &max_n);
    if (st != FCN_OK || a->num_frames == 0 || a->num_dets == 0) return st;
    cudaStream_t s = (cudaStream_t)stream;
    const int D = a->num_dets, F = a->num_frames;
    FCN_CUDA(fov_stage(w, a->num_points, D, F, max_n, a->scans, a->scan_offsets, a->frames, s));
    fx_count_kernel<<<D, FX_THREADS, 0, s>>>(F, a->scan_offsets, a->frames, a->boxes, a->det_frame, w.pos, w.fov_u,
                                             w.fov_v, a->det_points, w.keep, w.cnt, w.box, w.angle, w.bad);
    FCN_LAUNCH_CHECK();
    FCN_CUDA(job_totals(w, D, a->info, s));
    return FCN_OK;
}

extern "C" int fcn_frustum_extract_write(const fcn_frustum_extract_args *a, fcn_stream_t stream) {
    FxWs w;
    int max_n;
    const int st = fx_prepare(a, __func__, w, &max_n);
    if (st != FCN_OK || a->num_frames == 0 || a->num_dets == 0) return st;
    if (a->num_kept < 0 || a->num_kept > a->num_dets || a->num_out_points < 0 || a->num_out_points > INT32_MAX)
        return invalid(__func__, "num_kept must be in [0, num_dets] and num_out_points in [0, 2^31)");
    if (!a->offsets || (a->num_kept > 0 && (!a->frustum_angle || !a->box2d || !a->P || !a->det_index)) ||
        (a->num_out_points > 0 && !a->points))
        return invalid(__func__, "NULL output");
    cudaStream_t s = (cudaStream_t)stream;
    FCN_CUDA(cudaMemsetAsync(a->offsets, 0, 4, s));
    if (a->num_kept == 0) return FCN_OK;
    fx_write_kernel<<<a->num_dets, FX_THREADS, 0, s>>>(
        a->num_kept, a->num_out_points, a->scan_offsets, a->frames, a->det_frame, a->det_points, w.keep_pos,
        w.cnt_pos, w.box, w.angle, w.pos, w.fov_pts, w.fov_u, w.fov_v, (float4 *)a->points, a->offsets,
        a->frustum_angle, a->box2d, a->P, a->det_index);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}
