// KITTI refinement frustums on the device (C ABI section (16)): the three extraction functions of
// kitti/prepare_data_refine.py (:239-403 ground truth, :406-592 matched detections, :649-773 detections) for several
// frames and all their 3-D boxes in one pair of calls.
//
// The reference re-reads and re-projects every scan and runs one scipy Delaunay per box and augmentation.  Here the
// per-box constants (enlargement, perturbation, corners, angles) come from the host, and:
//   fcn_refine_extract_count  flags    the in-image test of every scan point (frustum_fov.cu, as section (15));
//                             scan     exclusive sum of the flags over all frames: the position of every in-image point;
//                             compact  the in-image points as float32 rect x, y, z and intensity, in scan order;
//                             iou      matched mode: one thread per (detection, ground truth) pair of a frame, the
//                                      standup-box pre-filter and the rotated 3-D IoU of rbbox_iou_3d in float64;
//                             match    matched mode: one thread per detection, the first maximum over its pairs and
//                                      the threshold test;
//                             count    one CTA per job over its frame's in-image points (L2-resident): the points in
//                                      the enlarged box, those also in the label box, and the drop rules;
//                             scans    exclusive sums over the kept jobs and their point counts, then info;
//   fcn_refine_extract_write  write    one CTA per kept job: the box tests again, a block scan for stable positions,
//                                      the points and their labels scattered in scan order.  Which job each kept
//                                      frustum is follows from job_points (the kept jobs in job order); the host has it.
#include <cmath>

#include "box_contains.cuh"
#include "box_iou.cuh"
#include "common.cuh"
#include "frame_refine.cuh"
#include "frustum_fov.cuh"

namespace fcn {

// bbox_overlaps_3d (ops/pybind11/rbbox_iou.py:62-96) of the two boxes' axis-aligned standup boxes, in its order
__device__ double rx_standup_iou(const double *__restrict__ c, const double *__restrict__ q) {
    double lo[2][3], hi[2][3];
    const double *b[2] = {c, q};
    for (int k = 0; k < 2; ++k)
        for (int a = 0; a < 3; ++a) {
            double mn = b[k][a], mx = b[k][a];
            for (int i = 1; i < 8; ++i) {
                const double v = b[k][3 * i + a];
                mn = v < mn ? v : mn;
                mx = v > mx ? v : mx;
            }
            lo[k][a] = mn;
            hi[k][a] = mx;
        }
    double vol[2], ext[3];
    for (int k = 0; k < 2; ++k)              // (x extent * z extent) * y extent
        vol[k] = __dmul_rn(__dmul_rn(__dsub_rn(hi[k][0], lo[k][0]), __dsub_rn(hi[k][2], lo[k][2])),
                           __dsub_rn(hi[k][1], lo[k][1]));
    const int axis[3] = {0, 2, 1};
    for (int i = 0; i < 3; ++i) {
        const int a = axis[i];
        const double e = __dsub_rn(fmin(hi[0][a], hi[1][a]), fmax(lo[0][a], lo[1][a]));
        ext[i] = e < 0.0 ? 0.0 : e;
    }
    const double inter = __dmul_rn(__dmul_rn(ext[0], ext[1]), ext[2]);
    return inter / __dsub_rn(__dadd_rn(vol[0], vol[1]), inter);
}

// the detection of pair t: the last d with pair_offsets[d] <= t
__device__ __forceinline__ int rx_det_of(const int32_t *__restrict__ po, int num_dets, int t) {
    int lo = 0, hi = num_dets - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (po[mid] <= t) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(FX_THREADS)
rx_iou_kernel(int num_pairs, int num_dets, int num_frames, int num_gt, const double *__restrict__ det_corners,
              const double *__restrict__ gt_corners, const int32_t *__restrict__ det_frame,
              const int32_t *__restrict__ gt_offsets, const int32_t *__restrict__ po, double *__restrict__ iou,
              int32_t *__restrict__ bad) {
    const int t = blockIdx.x * FX_THREADS + threadIdx.x;
    if (t >= num_pairs) return;
    const int d = rx_det_of(po, num_dets, t), f = det_frame[d];
    const int g = (f >= 0 && f < num_frames) ? gt_offsets[f] + (t - po[d]) : -1;
    if (g < 0 || g >= num_gt || (f >= 0 && f < num_frames && g >= gt_offsets[f + 1])) {
        iou[t] = 0.0;
        atomicAdd(bad, 1);
        return;
    }
    const double *c = det_corners + (size_t)d * 24, *q = gt_corners + (size_t)g * 24;
    iou[t] = rx_standup_iou(c, q) <= 0.0 ? 0.0 : rbbox_iou3d_d(c, q);
}

// overlap.max(0), overlap.argmax(0) (numpy: a NaN is the maximum, the first one wins) and `max < thresh -> skip`
__global__ void __launch_bounds__(FX_THREADS)
rx_match_kernel(int num_dets, int num_frames, double thresh, const int32_t *__restrict__ det_frame,
                const int32_t *__restrict__ gt_offsets, const int32_t *__restrict__ po,
                const double *__restrict__ iou, int32_t *__restrict__ match) {
    const int d = blockIdx.x * FX_THREADS + threadIdx.x;
    if (d >= num_dets) return;
    const int f = det_frame[d];
    if (f < 0 || f >= num_frames) {            // counted as bad by rx_iou_kernel when it has pairs
        match[d] = -1;
        return;
    }
    const int p0 = po[d], p1 = po[d + 1];
    int arg = -1;
    double best = 0.0;
    for (int p = p0; p < p1; ++p) {
        const double v = iou[p];
        if (isnan(v)) {
            arg = p - p0;
            best = v;
            break;
        }
        if (arg < 0 || v > best) {
            arg = p - p0;
            best = v;
        }
    }
    match[d] = (arg < 0 || best < thresh) ? -1 : gt_offsets[f] + arg;
}

// rx_count_kernel and rx_write_kernel keep their own loops and guards rather than job_count, job_words, kept_slot and
// job_scatter of frustum_fov.cuh: with those, ptxas schedules these two kernels differently.
__global__ void __launch_bounds__(FX_THREADS)
rx_count_kernel(int mode, int num_frames, int num_gt, int num_dets, const int32_t *__restrict__ so,
                const fcn_refine_box *__restrict__ jobs, const int32_t *__restrict__ job_frame,
                const int32_t *__restrict__ job_ref, const fcn_refine_box *__restrict__ gt_boxes,
                const int32_t *__restrict__ match, const int32_t *__restrict__ pos, const float4 *__restrict__ fov_pts,
                int32_t *__restrict__ job_points, int32_t *__restrict__ job_gt, int32_t *__restrict__ keep,
                long long *__restrict__ cnt, int32_t *__restrict__ bad) {
    using Reduce = cub::BlockReduce<int, FX_THREADS>;
    __shared__ typename Reduce::TempStorage tmp;
    const int j = blockIdx.x, f = job_frame[j];
    int g = -1;
    bool ok = f >= 0 && f < num_frames;
    if (mode == FCN_REFINE_GT) {
        g = job_ref[j];
        ok = ok && g >= 0 && g < num_gt;
    } else if (mode == FCN_REFINE_MATCHED) {
        const int d = job_ref[j];
        ok = ok && d >= 0 && d < num_dets;
        g = ok ? match[d] : -1;
    }
    if (!ok || (mode == FCN_REFINE_MATCHED && g < 0)) {
        if (threadIdx.x == 0) {
            job_points[j] = -1;
            job_gt[j] = -1;
            keep[j] = 0;
            cnt[j] = 0;
            if (!ok) atomicAdd(bad, 1);
        }
        return;
    }
    const fcn_refine_box box = jobs[j];
    fcn_refine_box lab;
    if (g >= 0) lab = gt_boxes[g];
    const int p0 = pos[so[f]], p1 = pos[so[f + 1]];
    int c = 0, l = 0;
    for (int i = p0 + threadIdx.x; i < p1; i += FX_THREADS) {
        const float4 p = fov_pts[i];
        if (box3d_contains(box, p)) {
            ++c;
            if (g >= 0) l += box3d_contains(lab, p);
        }
    }
    c = Reduce(tmp).Sum(c);
    __syncthreads();
    l = Reduce(tmp).Sum(l);
    if (threadIdx.x == 0) {
        const bool drop = mode == FCN_REFINE_DET ? c < 1 : l == 0;
        job_points[j] = drop ? -1 : c;
        job_gt[j] = g;
        keep[j] = drop ? 0 : 1;
        cnt[j] = drop ? 0 : c;
    }
}

__global__ void __launch_bounds__(FX_THREADS)
rx_write_kernel(int num_kept, long long num_out, const int32_t *__restrict__ so,
                const fcn_refine_box *__restrict__ jobs, const int32_t *__restrict__ job_frame,
                const fcn_refine_box *__restrict__ gt_boxes, const int32_t *__restrict__ job_points,
                const int32_t *__restrict__ job_gt, const int32_t *__restrict__ keep_pos,
                const long long *__restrict__ cnt_pos, const int32_t *__restrict__ pos,
                const float4 *__restrict__ fov_pts, float4 *__restrict__ points, uint8_t *__restrict__ labels,
                int32_t *__restrict__ offsets) {
    using Scan = cub::BlockScan<int, FX_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    const int j = blockIdx.x, c = job_points[j];
    if (c < 0) return;
    const int k = keep_pos[j];
    const long long base = cnt_pos[j];
    if (k >= num_kept || base + c > num_out) return;     // sizes read by the host disagree with the count pass
    const int f = job_frame[j], g = job_gt[j];
    if (threadIdx.x == 0) offsets[k + 1] = (int32_t)(base + c);
    const fcn_refine_box box = jobs[j];
    fcn_refine_box lab;
    const bool with_labels = labels != nullptr && g >= 0;
    if (with_labels) lab = gt_boxes[g];
    const int p0 = pos[so[f]], p1 = pos[so[f + 1]];
    int run = 0;
    for (int i0 = p0; i0 < p1 && run < c; i0 += FX_THREADS) {
        const int i = i0 + threadIdx.x;
        float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i < p1) p = fov_pts[i];
        const int flag = i < p1 && box3d_contains(box, p);
        int off, total;
        Scan(tmp).ExclusiveSum(flag, off, total);
        if (flag) {
            points[base + run + off] = p;
            if (with_labels) labels[base + run + off] = box3d_contains(lab, p) ? 1 : 0;
        }
        run += total;
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ host side
cudaError_t rx_count_det(int num_frames, int num_jobs, const int32_t *so, const fcn_refine_box *jobs,
                         const int32_t *job_frame, const int32_t *pos, const float4 *fov_pts, int32_t *job_points,
                         int32_t *job_gt, int32_t *keep, long long *cnt, int32_t *bad, cudaStream_t s) {
    rx_count_kernel<<<num_jobs, FX_THREADS, 0, s>>>(FCN_REFINE_DET, num_frames, 0, 0, so, jobs, job_frame, nullptr,
                                                    nullptr, nullptr, pos, fov_pts, job_points, job_gt, keep, cnt,
                                                    bad);
    return cudaGetLastError();
}

cudaError_t rx_write_det(int num_jobs, int num_kept, long long num_out, const int32_t *so, const fcn_refine_box *jobs,
                         const int32_t *job_frame, const int32_t *job_points, const int32_t *job_gt,
                         const int32_t *keep_pos, const long long *cnt_pos, const int32_t *pos, const float4 *fov_pts,
                         float4 *points, int32_t *offsets, cudaStream_t s) {
    rx_write_kernel<<<num_jobs, FX_THREADS, 0, s>>>(num_kept, num_out, so, jobs, job_frame, nullptr, job_points, job_gt,
                                                    keep_pos, cnt_pos, pos, fov_pts, points, nullptr, offsets);
    return cudaGetLastError();
}

struct RxWs : FovWs {
    double *iou;
    int32_t *match;
};

static cudaError_t rx_layout(const fcn_refine_extract_args *a, Carve &c, RxWs &w) {
    const cudaError_t e = fov_carve(c, a->num_points, a->num_jobs, false, w);
    const bool matched = a->mode == FCN_REFINE_MATCHED;
    w.iou = (double *)c.take(matched ? (size_t)a->num_pairs * 8 : 0);
    w.match = (int32_t *)c.take(matched ? (size_t)a->num_dets * 4 : 0);
    return e;
}

static bool rx_empty(const fcn_refine_extract_args *a) { return a->num_frames == 0 || a->num_jobs == 0; }

// Host-side checks shared by every entry: mode, counts, pointers, the scans.  Sets *max_n to the largest scan.
static int rx_check(const fcn_refine_extract_args *a, const char *fn, int *max_n) {
    if (a == nullptr) return invalid(fn, "NULL args");
    if (a->mode != FCN_REFINE_GT && a->mode != FCN_REFINE_MATCHED && a->mode != FCN_REFINE_DET)
        return invalid(fn, "mode must be FCN_REFINE_GT, FCN_REFINE_MATCHED or FCN_REFINE_DET");
    if (a->num_frames < 0 || a->num_points < 0 || a->num_jobs < 0 || a->num_gt < 0 || a->num_dets < 0 ||
        a->num_pairs < 0)
        return invalid(fn, "negative count");
    if (a->num_frames > 65535 || a->num_points > (1 << 30) || a->num_jobs > (1 << 28) || a->num_gt > (1 << 28) ||
        a->num_dets > (1 << 28) || a->num_pairs > (1 << 30))
        return invalid(fn, "too large (num_frames <= 65535, num_points, num_pairs <= 2^30, num_jobs, num_gt, "
                           "num_dets <= 2^28)");
    *max_n = 0;
    if (rx_empty(a)) return FCN_OK;
    if (!a->scan_offsets || !a->frames || !a->jobs || !a->job_frame || (a->num_points > 0 && !a->scans))
        return invalid(fn, "NULL pointer");
    if (a->mode != FCN_REFINE_DET && (!a->job_ref || (a->num_gt > 0 && !a->gt_boxes)))
        return invalid(fn, "NULL job_ref or gt_boxes");
    if (a->mode == FCN_REFINE_MATCHED &&
        (a->num_dets == 0 || !a->det_frame || !a->gt_offsets || !a->pair_offsets ||
         (a->num_pairs > 0 && (!a->gt_corners || !a->det_corners))))
        return invalid(fn, "matched mode needs num_dets > 0 and det_frame, gt_offsets, pair_offsets and corners");
    return check_scans(fn, a->host_scan_offsets, a->num_frames, a->num_points, a->scans, 16, max_n);
}

static int rx_prepare(const fcn_refine_extract_args *a, const char *fn, RxWs &w, int *max_n) {
    const int st = rx_check(a, fn, max_n);
    if (st != FCN_OK || rx_empty(a)) return st;
    if (!a->workspace || !a->info || !a->job_points || !a->job_gt)
        return invalid(fn, "NULL workspace, info, job_points or job_gt");
    return carve_workspace(fn, "refine_extract", a->workspace, a->workspace_bytes,
                           [&](Carve &c) { return rx_layout(a, c, w); });
}

}  // namespace fcn

using namespace fcn;

extern "C" long long fcn_refine_extract_workspace_bytes(const fcn_refine_extract_args *a) {
    int max_n;
    if (rx_check(a, __func__, &max_n) != FCN_OK) return -1;
    if (rx_empty(a)) return 0;
    RxWs w;
    return workspace_size(__func__, [&](Carve &c) { return rx_layout(a, c, w); });
}

extern "C" int fcn_refine_extract_count(const fcn_refine_extract_args *a, fcn_stream_t stream) {
    RxWs w;
    int max_n;
    const int st = rx_prepare(a, __func__, w, &max_n);
    if (st != FCN_OK || rx_empty(a)) return st;
    cudaStream_t s = (cudaStream_t)stream;
    const int J = a->num_jobs, F = a->num_frames;
    FCN_CUDA(fov_stage(w, a->num_points, J, F, max_n, a->scans, a->scan_offsets, a->frames, s));
    if (a->mode == FCN_REFINE_MATCHED) {
        if (a->num_pairs > 0) {
            rx_iou_kernel<<<ceil_div(a->num_pairs, FX_THREADS), FX_THREADS, 0, s>>>(
                a->num_pairs, a->num_dets, F, a->num_gt, a->det_corners, a->gt_corners, a->det_frame, a->gt_offsets,
                a->pair_offsets, w.iou, w.bad);
            FCN_LAUNCH_CHECK();
        }
        rx_match_kernel<<<ceil_div(a->num_dets, FX_THREADS), FX_THREADS, 0, s>>>(
            a->num_dets, F, a->iou_thresh, a->det_frame, a->gt_offsets, a->pair_offsets, w.iou, w.match);
        FCN_LAUNCH_CHECK();
    }
    rx_count_kernel<<<J, FX_THREADS, 0, s>>>(a->mode, F, a->num_gt, a->num_dets, a->scan_offsets, a->jobs,
                                             a->job_frame, a->job_ref, a->gt_boxes, w.match, w.pos, w.fov_pts,
                                             a->job_points, a->job_gt, w.keep, w.cnt, w.bad);
    FCN_LAUNCH_CHECK();
    FCN_CUDA(job_totals(w, J, a->info, s));
    return FCN_OK;
}

extern "C" int fcn_refine_extract_write(const fcn_refine_extract_args *a, fcn_stream_t stream) {
    RxWs w;
    int max_n;
    const int st = rx_prepare(a, __func__, w, &max_n);
    if (st != FCN_OK || rx_empty(a)) return st;
    if (a->num_kept < 0 || a->num_kept > a->num_jobs || a->num_out_points < 0 || a->num_out_points > INT32_MAX)
        return invalid(__func__, "num_kept must be in [0, num_jobs] and num_out_points in [0, 2^31)");
    if (!a->offsets || (a->num_out_points > 0 && !a->points))
        return invalid(__func__, "NULL output");
    cudaStream_t s = (cudaStream_t)stream;
    FCN_CUDA(cudaMemsetAsync(a->offsets, 0, 4, s));
    if (a->num_kept == 0) return FCN_OK;
    uint8_t *labels = a->mode == FCN_REFINE_DET ? nullptr : a->labels;
    rx_write_kernel<<<a->num_jobs, FX_THREADS, 0, s>>>(
        a->num_kept, a->num_out_points, a->scan_offsets, a->jobs, a->job_frame, a->gt_boxes, a->job_points, a->job_gt,
        w.keep_pos, w.cnt_pos, w.pos, w.fov_pts, (float4 *)a->points, labels, a->offsets);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}
