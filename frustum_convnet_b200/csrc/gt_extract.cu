// KITTI first-stage training frustums on the device (C ABI section (17)): the point work of extract_frustum_data and
// extract_frustum_det_data (kitti/prepare_data.py:260-391 and :102-257) for several frames and all their jobs in one
// pair of calls.  A job is one cutting 2-D box and one label 3-D box in one frame.
//
// The reference re-projects every scan and runs one scipy Delaunay per box and augmentation.  Here the perturbation,
// the 2-D matching and every per-box constant come from the host, and:
//   fcn_gt_extract_count  flags    the in-image test of every scan point (frustum_fov.cuh, as section (15));
//                         scan     exclusive sum of the flags over all frames: the position of every in-image point;
//                         compact  the in-image points as float32 rect x, y, z and intensity plus float64 u, v;
//                         count    one CTA per job over its frame's in-image points (L2-resident): the points in the
//                                  unclipped cutting box (:324-328), those also in the label box (box_contains.cuh),
//                                  and the drop rule (no labelled point, :354);
//                         scans    exclusive sums over the kept jobs and their point counts, then info;
//   fcn_gt_extract_write  write    one CTA per kept job: the box tests again, a block scan for stable positions, the
//                                  points and their labels scattered in scan order.
#include <cub/cub.cuh>

#include <cmath>

#include "box_contains.cuh"
#include "common.cuh"
#include "frustum_fov.cuh"

namespace fcn {

__global__ void __launch_bounds__(FX_THREADS)
gx_flag_kernel(const float4 *__restrict__ scans, const int32_t *__restrict__ so,
               const fcn_frustum_frame *__restrict__ frames, int32_t *__restrict__ flags) {
    fov_flag(scans, so, frames, flags);
}

__global__ void __launch_bounds__(FX_THREADS)
gx_compact_kernel(const float4 *__restrict__ scans, const int32_t *__restrict__ so,
                  const fcn_frustum_frame *__restrict__ frames, const int32_t *__restrict__ pos,
                  float4 *__restrict__ fov_pts, double *__restrict__ fov_u, double *__restrict__ fov_v) {
    fov_compact<true>(scans, so, frames, pos, fov_pts, fov_u, fov_v);
}

// prepare_data.py:324-327, in its order: u < xmax, u >= xmin, v < ymax, v >= ymin
__device__ __forceinline__ bool gx_in_box2d(double u, double v, const fcn_gt_job &jb) {
    return u < jb.box[2] && u >= jb.box[0] && v < jb.box[3] && v >= jb.box[1];
}

__global__ void __launch_bounds__(FX_THREADS)
gx_count_kernel(int num_frames, int num_labels, const int32_t *__restrict__ so, const fcn_gt_job *__restrict__ jobs,
                const fcn_refine_box *__restrict__ label_boxes, const int32_t *__restrict__ pos,
                const float4 *__restrict__ fov_pts, const double *__restrict__ fov_u,
                const double *__restrict__ fov_v, int32_t *__restrict__ job_points, int32_t *__restrict__ keep,
                long long *__restrict__ cnt, int32_t *__restrict__ bad) {
    using Reduce = cub::BlockReduce<int, FX_THREADS>;
    __shared__ typename Reduce::TempStorage tmp;
    const int j = blockIdx.x;
    const fcn_gt_job jb = jobs[j];
    const int f = jb.frame, g = jb.label;
    if (f < 0 || f >= num_frames || g < 0 || g >= num_labels) {
        if (threadIdx.x == 0) {
            job_points[j] = -1;
            keep[j] = 0;
            cnt[j] = 0;
            atomicAdd(bad, 1);
        }
        return;
    }
    const fcn_refine_box lab = label_boxes[g];
    const int p0 = pos[so[f]], p1 = pos[so[f + 1]];
    int c = 0, l = 0;
    for (int i = p0 + threadIdx.x; i < p1; i += FX_THREADS) {
        if (gx_in_box2d(fov_u[i], fov_v[i], jb)) {
            ++c;
            l += box3d_contains(lab, fov_pts[i]);
        }
    }
    c = Reduce(tmp).Sum(c);
    __syncthreads();
    l = Reduce(tmp).Sum(l);
    if (threadIdx.x == 0) {
        const bool drop = l == 0;
        job_points[j] = drop ? -1 : c;
        keep[j] = drop ? 0 : 1;
        cnt[j] = drop ? 0 : c;
    }
}

__global__ void gx_info_kernel(int num_jobs, const int32_t *__restrict__ keep_pos,
                               const long long *__restrict__ cnt_pos, const int32_t *__restrict__ bad,
                               long long *__restrict__ info) {
    info[0] = keep_pos[num_jobs];
    info[1] = cnt_pos[num_jobs];
    info[2] = *bad;
    info[3] = 0;
}

__global__ void __launch_bounds__(FX_THREADS)
gx_write_kernel(int num_kept, long long num_out, const int32_t *__restrict__ so, const fcn_gt_job *__restrict__ jobs,
                const fcn_refine_box *__restrict__ label_boxes, const int32_t *__restrict__ job_points,
                const int32_t *__restrict__ keep_pos, const long long *__restrict__ cnt_pos,
                const int32_t *__restrict__ pos, const float4 *__restrict__ fov_pts, const double *__restrict__ fov_u,
                const double *__restrict__ fov_v, float4 *__restrict__ points, uint8_t *__restrict__ labels,
                int32_t *__restrict__ offsets) {
    using Scan = cub::BlockScan<int, FX_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    const int j = blockIdx.x, c = job_points[j];
    if (c < 0) return;
    const int k = keep_pos[j];
    const long long base = cnt_pos[j];
    if (k >= num_kept || base + c > num_out) return;     // sizes read by the host disagree with the count pass
    if (threadIdx.x == 0) offsets[k + 1] = (int32_t)(base + c);
    const fcn_gt_job jb = jobs[j];
    const fcn_refine_box lab = label_boxes[jb.label];
    const int p0 = pos[so[jb.frame]], p1 = pos[so[jb.frame + 1]];
    int run = 0;
    for (int i0 = p0; i0 < p1 && run < c; i0 += FX_THREADS) {
        const int i = i0 + threadIdx.x;
        const int flag = i < p1 && gx_in_box2d(fov_u[i], fov_v[i], jb);
        int off, total;
        Scan(tmp).ExclusiveSum(flag, off, total);
        if (flag) {
            const float4 p = fov_pts[i];
            points[base + run + off] = p;
            labels[base + run + off] = box3d_contains(lab, p) ? 1 : 0;
        }
        run += total;
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ host side
struct GxWs {
    int32_t *flags, *pos, *keep, *keep_pos, *bad;
    long long *cnt, *cnt_pos;
    float4 *fov_pts;
    double *fov_u, *fov_v;
    void *temp;
    size_t temp_bytes;
};

static cudaError_t gx_layout(const fcn_gt_extract_args *a, Carve &c, GxWs &w) {
    const size_t N = (size_t)a->num_points, J = (size_t)a->num_jobs;
    size_t t0 = 0, t1 = 0, t2 = 0;
    cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, t0, (const int32_t *)nullptr, (int32_t *)nullptr,
                                                  a->num_points + 1);
    if (e != cudaSuccess) return e;
    e = cub::DeviceScan::ExclusiveSum(nullptr, t1, (const int32_t *)nullptr, (int32_t *)nullptr, a->num_jobs + 1);
    if (e != cudaSuccess) return e;
    e = cub::DeviceScan::ExclusiveSum(nullptr, t2, (const long long *)nullptr, (long long *)nullptr,
                                      a->num_jobs + 1);
    if (e != cudaSuccess) return e;
    w.temp_bytes = t0 > t1 ? t0 : t1;
    w.temp_bytes = w.temp_bytes > t2 ? w.temp_bytes : t2;
    w.flags = (int32_t *)c.take((N + 1) * 4);
    w.pos = (int32_t *)c.take((N + 1) * 4);
    w.fov_pts = (float4 *)c.take(N * 16);
    w.fov_u = (double *)c.take(N * 8);
    w.fov_v = (double *)c.take(N * 8);
    w.keep = (int32_t *)c.take((J + 1) * 4);
    w.keep_pos = (int32_t *)c.take((J + 1) * 4);
    w.cnt = (long long *)c.take((J + 1) * 8);
    w.cnt_pos = (long long *)c.take((J + 1) * 8);
    w.bad = (int32_t *)c.take(4);
    w.temp = c.take(w.temp_bytes);
    return cudaSuccess;
}

static bool gx_empty(const fcn_gt_extract_args *a) { return a->num_frames == 0 || a->num_jobs == 0; }

// Host-side checks shared by every entry: counts, pointers, the scans.  Sets *max_n to the largest scan.
static int gx_check(const fcn_gt_extract_args *a, const char *fn, int *max_n) {
    if (a == nullptr) return invalid(fn, "NULL args");
    if (a->num_frames < 0 || a->num_points < 0 || a->num_jobs < 0 || a->num_labels < 0)
        return invalid(fn, "negative count (num_frames, num_points, num_jobs, num_labels must be >= 0)");
    if (a->num_frames > 65535 || a->num_points > (1 << 30) || a->num_jobs > (1 << 28) || a->num_labels > (1 << 28))
        return invalid(fn, "too large (num_frames <= 65535, num_points <= 2^30, num_jobs, num_labels <= 2^28)");
    *max_n = 0;
    if (gx_empty(a)) return FCN_OK;
    if (!a->scan_offsets || !a->frames || !a->jobs || (a->num_labels > 0 && !a->label_boxes) ||
        (a->num_points > 0 && !a->scans))
        return invalid(fn, "NULL pointer");
    return check_scans(fn, a->host_scan_offsets, a->num_frames, a->num_points, a->scans, max_n);
}

static int gx_prepare(const fcn_gt_extract_args *a, const char *fn, GxWs &w, int *max_n) {
    const int st = gx_check(a, fn, max_n);
    if (st != FCN_OK || gx_empty(a)) return st;
    if (!a->workspace || !a->info || !a->job_points) return invalid(fn, "NULL workspace, info or job_points");
    return carve_workspace(fn, "gt_extract", a->workspace, a->workspace_bytes,
                           [&](Carve &c) { return gx_layout(a, c, w); });
}

}  // namespace fcn

using namespace fcn;

extern "C" long long fcn_gt_extract_workspace_bytes(const fcn_gt_extract_args *a) {
    int max_n;
    if (gx_check(a, __func__, &max_n) != FCN_OK) return -1;
    if (gx_empty(a)) return 0;
    GxWs w;
    return workspace_size(__func__, [&](Carve &c) { return gx_layout(a, c, w); });
}

extern "C" int fcn_gt_extract_count(const fcn_gt_extract_args *a, fcn_stream_t stream) {
    GxWs w;
    int max_n;
    const int st = gx_prepare(a, __func__, w, &max_n);
    if (st != FCN_OK || gx_empty(a)) return st;
    cudaStream_t s = (cudaStream_t)stream;
    const int N = a->num_points, J = a->num_jobs, F = a->num_frames;
    const float4 *scans = (const float4 *)a->scans;
    FCN_CUDA(cudaMemsetAsync(w.flags + N, 0, 4, s));
    FCN_CUDA(cudaMemsetAsync(w.keep + J, 0, 4, s));
    FCN_CUDA(cudaMemsetAsync(w.cnt + J, 0, 8, s));
    FCN_CUDA(cudaMemsetAsync(w.bad, 0, 4, s));
    const dim3 grid(ceil_div(max_n, FX_THREADS), F);
    if (max_n > 0) {
        gx_flag_kernel<<<grid, FX_THREADS, 0, s>>>(scans, a->scan_offsets, a->frames, w.flags);
        FCN_LAUNCH_CHECK();
    }
    FCN_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, w.temp_bytes, w.flags, w.pos, N + 1, s));
    if (max_n > 0) {
        gx_compact_kernel<<<grid, FX_THREADS, 0, s>>>(scans, a->scan_offsets, a->frames, w.pos, w.fov_pts, w.fov_u,
                                                      w.fov_v);
        FCN_LAUNCH_CHECK();
    }
    gx_count_kernel<<<J, FX_THREADS, 0, s>>>(F, a->num_labels, a->scan_offsets, a->jobs, a->label_boxes, w.pos,
                                             w.fov_pts, w.fov_u, w.fov_v, a->job_points, w.keep, w.cnt, w.bad);
    FCN_LAUNCH_CHECK();
    FCN_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, w.temp_bytes, w.keep, w.keep_pos, J + 1, s));
    FCN_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, w.temp_bytes, w.cnt, w.cnt_pos, J + 1, s));
    gx_info_kernel<<<1, 1, 0, s>>>(J, w.keep_pos, w.cnt_pos, w.bad, a->info);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

extern "C" int fcn_gt_extract_write(const fcn_gt_extract_args *a, fcn_stream_t stream) {
    GxWs w;
    int max_n;
    const int st = gx_prepare(a, __func__, w, &max_n);
    if (st != FCN_OK || gx_empty(a)) return st;
    if (a->num_kept < 0 || a->num_kept > a->num_jobs || a->num_out_points < 0 || a->num_out_points > INT32_MAX)
        return invalid(__func__, "num_kept must be in [0, num_jobs] and num_out_points in [0, 2^31)");
    if (!a->offsets || (a->num_out_points > 0 && (!a->points || !a->labels)))
        return invalid(__func__, "NULL output");
    cudaStream_t s = (cudaStream_t)stream;
    FCN_CUDA(cudaMemsetAsync(a->offsets, 0, 4, s));
    if (a->num_kept == 0) return FCN_OK;
    gx_write_kernel<<<a->num_jobs, FX_THREADS, 0, s>>>(
        a->num_kept, a->num_out_points, a->scan_offsets, a->jobs, a->label_boxes, a->job_points, w.keep_pos,
        w.cnt_pos, w.pos, w.fov_pts, w.fov_u, w.fov_v, (float4 *)a->points, a->labels, a->offsets);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}
