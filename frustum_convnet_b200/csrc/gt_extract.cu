// KITTI first-stage training frustums on the device (C ABI section (17)): the point work of extract_frustum_data and
// extract_frustum_det_data (kitti/prepare_data.py:260-391 and :102-257) for several frames and all their jobs in one
// pair of calls.  A job is one cutting 2-D box and one label 3-D box in one frame.
//
// The reference re-projects every scan and runs one scipy Delaunay per box and augmentation.  Here the perturbation,
// the 2-D matching and every per-box constant come from the host, and:
//   fcn_gt_extract_count  flags    the in-image test of every scan point (frustum_fov.cu, as section (15));
//                         scan     exclusive sum of the flags over all frames: the position of every in-image point;
//                         compact  the in-image points as float32 rect x, y, z and intensity plus float64 u, v;
//                         count    one CTA per job over its frame's in-image points (L2-resident): the points in the
//                                  unclipped cutting box (:324-328), those also in the label box (box_contains.cuh),
//                                  and the drop rule (no labelled point, :354);
//                         scans    exclusive sums over the kept jobs and their point counts, then info;
//   fcn_gt_extract_write  write    one CTA per kept job: the box tests again, a block scan for stable positions, the
//                                  points and their labels scattered in scan order.
#include <cmath>

#include "box_contains.cuh"
#include "common.cuh"
#include "frustum_fov.cuh"

namespace fcn {

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
    const int j = blockIdx.x;
    const fcn_gt_job jb = jobs[j];
    const int f = jb.frame, g = jb.label;
    if (f < 0 || f >= num_frames || g < 0 || g >= num_labels) {
        if (threadIdx.x == 0) {
            job_words(j, true, 0, job_points, keep, cnt);
            atomicAdd(bad, 1);
        }
        return;
    }
    const fcn_refine_box lab = label_boxes[g];
    int c, l;
    job_count<true>(pos[so[f]], pos[so[f + 1]], c, l, [&](int i, int &c, int &l) {
        if (gx_in_box2d(fov_u[i], fov_v[i], jb)) {
            ++c;
            l += box3d_contains(lab, fov_pts[i]);
        }
    });
    if (threadIdx.x == 0) job_words(j, l == 0, c, job_points, keep, cnt);
}

__global__ void __launch_bounds__(FX_THREADS)
gx_write_kernel(int num_kept, long long num_out, const int32_t *__restrict__ so, const fcn_gt_job *__restrict__ jobs,
                const fcn_refine_box *__restrict__ label_boxes, const int32_t *__restrict__ job_points,
                const int32_t *__restrict__ keep_pos, const long long *__restrict__ cnt_pos,
                const int32_t *__restrict__ pos, const float4 *__restrict__ fov_pts, const double *__restrict__ fov_u,
                const double *__restrict__ fov_v, float4 *__restrict__ points, uint8_t *__restrict__ labels,
                int32_t *__restrict__ offsets) {
    const int j = blockIdx.x, c = job_points[j];
    int k;
    long long base;
    if (!kept_slot(j, c, num_kept, num_out, keep_pos, cnt_pos, offsets, &k, &base)) return;
    const fcn_gt_job jb = jobs[j];
    const fcn_refine_box lab = label_boxes[jb.label];
    job_scatter(pos[so[jb.frame]], pos[so[jb.frame + 1]], c, base,
                [&](int i) { return gx_in_box2d(fov_u[i], fov_v[i], jb); }, [&](long long o, int i) {
                    const float4 p = fov_pts[i];
                    points[o] = p;
                    labels[o] = box3d_contains(lab, p) ? 1 : 0;
                });
}

// ------------------------------------------------------------------------------------------------ host side
static cudaError_t gx_layout(const fcn_gt_extract_args *a, Carve &c, FovWs &w) {
    return fov_carve(c, a->num_points, a->num_jobs, true, w);
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
    return check_scans(fn, a->host_scan_offsets, a->num_frames, a->num_points, a->scans, 16, max_n);
}

static int gx_prepare(const fcn_gt_extract_args *a, const char *fn, FovWs &w, int *max_n) {
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
    FovWs w;
    return workspace_size(__func__, [&](Carve &c) { return gx_layout(a, c, w); });
}

extern "C" int fcn_gt_extract_count(const fcn_gt_extract_args *a, fcn_stream_t stream) {
    FovWs w;
    int max_n;
    const int st = gx_prepare(a, __func__, w, &max_n);
    if (st != FCN_OK || gx_empty(a)) return st;
    cudaStream_t s = (cudaStream_t)stream;
    const int J = a->num_jobs, F = a->num_frames;
    FCN_CUDA(fov_stage(w, a->num_points, J, F, max_n, a->scans, a->scan_offsets, a->frames, s));
    gx_count_kernel<<<J, FX_THREADS, 0, s>>>(F, a->num_labels, a->scan_offsets, a->jobs, a->label_boxes, w.pos,
                                             w.fov_pts, w.fov_u, w.fov_v, a->job_points, w.keep, w.cnt, w.bad);
    FCN_LAUNCH_CHECK();
    FCN_CUDA(job_totals(w, J, a->info, s));
    return FCN_OK;
}

extern "C" int fcn_gt_extract_write(const fcn_gt_extract_args *a, fcn_stream_t stream) {
    FovWs w;
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
