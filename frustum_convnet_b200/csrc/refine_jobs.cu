// The refinement stage's inputs from the detection collector's device rows (C ABI section (20)): the jobs of
// extract_frustum_data_rgb_detection and extract_frustum_det_data (kitti/prepare_data_refine.py:649-773, :406-592) for
// section (16)'s count and write passes, and the per-frustum lists and fcn_train_frustum records
// (datasets/provider_sample_refine.py:217-226, generate_ref :336-385) of the kept frustums, with no host pass over the
// rows.
//
//   fcn_refine_jobs_from_rows   one thread per job: its piece by binary search over piece_offsets (the host's gather
//                               plan), the row read back as write_detection_results' text, the box array, the checks,
//                               the x1.2 enlargement and the fcn_refine_box that rx_count_kernel / rx_write_kernel take;
//   fcn_refine_frustum_table    one thread per kept frustum: the corners, angles and records of the enlarged box.
//
// Exactness.  The quantization is det_quantize.cuh's.  Every float64 product and sum is __dmul_rn / __dadd_rn /
// __dsub_rn, or __fma_rn where numpy's np.dot goes through BLAS in the order OpenBLAS's kernels sum (dgemm: the first
// product rounded, then one fused multiply-add per further term; dgemv of a 2-vector: the second product rounded, then
// the first fused), so contraction cannot change them.  The centre-view box of generate_ref
// has angle 0 and centre 0, so its corners are exactly (+-l/2, +-h/2, +-w/2): its face means are (0, 0, -+w/2), its
// arange runs from -w/2 to w/2 and T = ceil(w / s), all exact (tests/test_refine_cascade_cpu.py restates this against
// train_inputs.refine_ref_line).  cos, sin and atan2 are CUDA's float64 functions (<= 2 ulp from glibc's).
#include <cmath>

#include "common.cuh"
#include "det_quantize.cuh"
#include "frame_refine.cuh"

namespace fcn {

constexpr int RJ_THREADS = 256;
constexpr double RJ_RATIO = 1.2;        // the enlargement of every box that cuts points (prepare_data_refine.py:724)

// the piece of job j: the last p with piece_offsets[p] <= j (empty pieces skipped)
__device__ __forceinline__ int rj_piece_of(const int32_t *__restrict__ off, int num_pieces, int j) {
    int lo = 0, hi = num_pieces - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= j) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// corner i of compute_box_3d's order: x = +-l/2, y = +-h/2, z = +-w/2 (half extents hl, hh, hw)
__device__ __forceinline__ void rj_corner(int i, double hl, double hh, double hw, double &xc, double &yc, double &zc) {
    xc = (i & 2) ? -hl : hl;                       // [1, 1, -1, -1, 1, 1, -1, -1]
    yc = i < 4 ? hh : -hh;                         // [1, 1, 1, 1, -1, -1, -1, -1]
    zc = ((i + 1) & 2) ? -hw : hw;                 // [1, -1, -1, 1, 1, -1, -1, 1]
}

__global__ void __launch_bounds__(RJ_THREADS) rj_jobs_kernel(fcn_refine_jobs_args a) {
    const int j = blockIdx.x * RJ_THREADS + threadIdx.x;
    if (j >= a.num_jobs) return;
    const int p = rj_piece_of(a.piece_offsets, a.num_pieces, j);
    const float *__restrict__ row = a.rows + (size_t)(a.piece_row[p] + (j - a.piece_offsets[p])) * 12;
    // row [x1, y1, x2, y2, tx, ty, tz, h, w, l, ry, score], each as utils.read_label reads its text back
    double b[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) b[i] = df_quantize(row[i], 1e4);
    const double tx = df_quantize(row[4], 1e4), ty = df_quantize(row[5], 1e4), tz = df_quantize(row[6], 1e4);
    const double h = df_quantize(row[7], 1e4), w = df_quantize(row[8], 1e4), l = df_quantize(row[9], 1e4);
    const double ry = df_quantize(row[10], 1e4), score = df_quantize(row[11], 1e6);
    const double box[7] = {tx, __dsub_rn(ty, __dmul_rn(h, 0.5)), tz, l, w, h, ry};      // obj_array
    int st = 0;
#pragma unroll
    for (int i = 0; i < 7; ++i)
        if (!isfinite(box[i])) st = FCN_REFINE_ROW_NONFINITE;
    if (!(l > 0.0 && w > 0.0 && h > 0.0)) st |= FCN_REFINE_ROW_EXTENTS;
    const bool det = a.mode == FCN_REFINE_DET;
    if (det && (__dsub_rn(b[3], b[1]) < 5.0 || __dsub_rn(b[2], b[0]) < 1.0)) st |= FCN_REFINE_ROW_DROPPED;
    a.status[j] = st;

    fcn_refine_job_data d;
    d.cut[0] = box[0];
    d.cut[1] = box[1];
    d.cut[2] = box[2];
    d.cut[3] = __dmul_rn(l, RJ_RATIO);
    d.cut[4] = __dmul_rn(w, RJ_RATIO);
    d.cut[5] = __dmul_rn(h, RJ_RATIO);
    d.cut[6] = ry;
#pragma unroll
    for (int i = 0; i < 4; ++i) d.box2d[i] = b[i];
    d.prob = score;
    d.image = a.piece_image[p];
    d.cls_index = a.piece_class[p];
    a.job_data[j] = d;

    fcn_refine_box r;                               // box_record of the enlarged box
    r.center[0] = d.cut[0];
    r.center[1] = d.cut[1];
    r.center[2] = d.cut[2];
    const bool cut = det && st != 0;                // no point is in it: the count pass drops the job
    r.half[0] = cut ? -1.0 : __dmul_rn(d.cut[3], 0.5);
    r.half[1] = cut ? -1.0 : __dmul_rn(d.cut[5], 0.5);
    r.half[2] = cut ? -1.0 : __dmul_rn(d.cut[4], 0.5);
    r.cs = cos(ry);
    r.sn = sin(ry);
    a.jobs[j] = r;
    a.job_frame[j] = a.piece_frame[p];
    a.job_ref[j] = j;
    if (a.mode != FCN_REFINE_MATCHED) return;
    // iou_corners (boxes3d2corners) of the box array: R @ corners with R = [[c, 0, s], [0, 1, 0], [-s, 0, c]], each
    // product rounded and summed in order (the zero terms add nothing), then the centre
    const double hl = __dmul_rn(l, 0.5), hh = __dmul_rn(h, 0.5), hw = __dmul_rn(w, 0.5);
    double *__restrict__ out = a.det_corners + (size_t)j * 24;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        double xc, yc, zc;
        rj_corner(i, hl, hh, hw, xc, yc, zc);
        out[3 * i + 0] = __dadd_rn(__dadd_rn(__dmul_rn(r.cs, xc), __dmul_rn(r.sn, zc)), box[0]);
        out[3 * i + 1] = __dadd_rn(yc, box[1]);
        out[3 * i + 2] = __dadd_rn(__dadd_rn(__dmul_rn(-r.sn, xc), __dmul_rn(r.cs, zc)), box[2]);
    }
}

__global__ void __launch_bounds__(RJ_THREADS) rj_table_kernel(fcn_refine_frustum_table_args a) {
    const int k = blockIdx.x * RJ_THREADS + threadIdx.x;
    if (k >= a.num_kept) return;
    const int j = a.kept[k];
    const fcn_refine_job_data d = a.job_data[j];
    const double *cut = d.cut;
    const double c = cos(cut[6]), s = sin(cut[6]);
    const double hl = __dmul_rn(cut[3], 0.5), hw = __dmul_rn(cut[4], 0.5), hh = __dmul_rn(cut[5], 0.5);
    double *__restrict__ L = a.lists + (size_t)k * FCN_REFINE_LIST_COLS;
    L[0] = -atan2(cut[2], cut[0]);                  // frustum_angle
    double p0[3], p6[3];
#pragma unroll
    for (int i = 0; i < 8; ++i) {                   // compute_box_3d_obj_array: np.dot(R, corners) (dgemm), + centre
        double xc, yc, zc;
        rj_corner(i, hl, hh, hw, xc, yc, zc);
        const double x = __dadd_rn(__fma_rn(s, zc, __dmul_rn(c, xc)), cut[0]);
        const double y = __dadd_rn(yc, cut[1]);
        const double z = __dadd_rn(__fma_rn(c, zc, __dmul_rn(-s, xc)), cut[2]);
        L[1 + 3 * i] = x;
        L[2 + 3 * i] = y;
        L[3 + 3 * i] = z;
        if (i == 0) p0[0] = x, p0[1] = y, p0[2] = z;
        if (i == 6) p6[0] = x, p6[1] = y, p6[2] = z;
    }
    L[25] = cut[3];
    L[26] = cut[4];
    L[27] = cut[5];
    L[28] = cut[6];
#pragma unroll
    for (int i = 0; i < 4; ++i) L[29 + i] = d.box2d[i];
    L[33] = d.prob;

    fcn_train_frustum *__restrict__ r = a.records + k;
    r->rot = cut[6];
    r->cs = c;
    r->sn = s;
    double pc[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        pc[i] = __dmul_rn(__dadd_rn(p0[i], p6[i]), 0.5);
        r->ref_center[i] = pc[i];
    }
    // refine_ref_line of the centre-view box (exact, see the top of the file)
    const double z1 = -hw;
    r->line0[0] = 0.0;
    r->line0[1] = 0.0;
    r->line0[2] = z1;
    r->line_delta[0] = 0.0;
    r->line_delta[1] = 0.0;
    r->line_delta[2] = __dsub_rn(hw, z1);
    r->z_start = z1;
    int32_t *__restrict__ wd = a.words + (size_t)k * (a.num_scales + 1);
    bool degenerate = !(r->line_delta[2] != 0.0);
    for (int q = 0; q < a.num_scales; ++q) {
        const double st = a.stride[q];
        r->z_step[q] = __dsub_rn(__dadd_rn(z1, st), z1);
        const double n = ceil(__ddiv_rn(__dsub_rn(hw, z1), st));       // len(np.arange(z1, z2, s))
        const int T = n > 0.0 ? (int)fmin(n, 2147483647.0) : 0;
        r->T[q] = T;
        wd[q] = T;
        degenerate = degenerate || T < 1;
    }
    wd[a.num_scales] = degenerate ? 1 : 0;
    r->cls_index = d.cls_index;
    if (!a.labels) {
        r->rgb_prob = d.prob;
        return;
    }
    // provider_sample_refine.py:141-147: the ground truth's centre minus the predicted centre, rotated by the
    // predicted angle (rotate_pc_along_y: np.dot of a row by the transposed rotation, which OpenBLAS's dgemv sums as
    // the second product rounded, then the first fused onto it), heading minus the angle
    const int g = a.job_gt[j];
    if (g < 0 || g >= a.num_gt) return;
    const fcn_refine_gt_terms t = a.gt_terms[g];
    const double dx = __dsub_rn(t.center[0], pc[0]), dy = __dsub_rn(t.center[1], pc[1]);
    const double dz = __dsub_rn(t.center[2], pc[2]);
    r->center[0] = __fma_rn(dx, c, __dmul_rn(dz, -s));
    r->center[1] = dy;
    r->center[2] = __fma_rn(dx, s, __dmul_rn(dz, c));
    r->heading = __dsub_rn(t.heading, cut[6]);
#pragma unroll
    for (int i = 0; i < 3; ++i) r->size[i] = t.size[i];
    r->dist = t.dist;
}

cudaError_t rj_jobs(const fcn_refine_jobs_args &a, cudaStream_t s) {
    rj_jobs_kernel<<<ceil_div(a.num_jobs, RJ_THREADS), RJ_THREADS, 0, s>>>(a);
    return cudaGetLastError();
}

cudaError_t rj_table(const fcn_refine_frustum_table_args &a, cudaStream_t s) {
    rj_table_kernel<<<ceil_div(a.num_kept, RJ_THREADS), RJ_THREADS, 0, s>>>(a);
    return cudaGetLastError();
}

// Host-side checks of the gather plan: counts, the host copies and pointers.
static int rj_check(const fcn_refine_jobs_args *a, const char *fn) {
    if (a == nullptr) return invalid(fn, "NULL args");
    if (a->mode != FCN_REFINE_MATCHED && a->mode != FCN_REFINE_DET)
        return invalid(fn, "mode must be FCN_REFINE_MATCHED or FCN_REFINE_DET");
    const int P = a->num_pieces;
    if (P < 0 || a->num_jobs < 0 || a->num_rows < 0) return invalid(fn, "negative count");
    if (a->num_jobs > (1 << 28)) return invalid(fn, "too many jobs (num_jobs <= 2^28)");
    if (!a->host_piece_offsets || !a->host_piece_row) return invalid(fn, "NULL host copies");
    if (!offsets_ok(a->host_piece_offsets, P, a->num_jobs))
        return invalid(fn, "piece_offsets must start at 0, never decrease and end at num_jobs");
    for (int p = 0; p < P; ++p) {
        const long long r0 = a->host_piece_row[p], n = a->host_piece_offsets[p + 1] - a->host_piece_offsets[p];
        if (r0 < 0 || r0 + n > a->num_rows) return invalid(fn, "a piece's rows must lie inside [0, num_rows)");
    }
    if (a->num_jobs == 0) return FCN_OK;
    if (!a->rows || !a->piece_offsets || !a->piece_row || !a->piece_frame || !a->piece_image || !a->piece_class ||
        !a->jobs || !a->job_frame || !a->job_ref || !a->status || !a->job_data ||
        (a->mode == FCN_REFINE_MATCHED && !a->det_corners))
        return invalid(fn, "NULL pointer");
    return FCN_OK;
}

static int rt_check(const fcn_refine_frustum_table_args *a, const char *fn) {
    if (a == nullptr) return invalid(fn, "NULL args");
    if (a->mode != FCN_REFINE_MATCHED && a->mode != FCN_REFINE_DET)
        return invalid(fn, "mode must be FCN_REFINE_MATCHED or FCN_REFINE_DET");
    if (a->num_kept < 0 || a->num_jobs < 0 || a->num_gt < 0 || a->num_kept > a->num_jobs)
        return invalid(fn, "counts must be >= 0 and num_kept <= num_jobs");
    if (a->num_scales < 1 || a->num_scales > FCN_MAX_SCALES) return invalid(fn, "num_scales must be in [1, 8]");
    for (int q = 0; q < a->num_scales; ++q)
        if (!(a->stride[q] > 0.0) || !std::isfinite(a->stride[q])) return invalid(fn, "strides must be positive");
    if (a->labels && a->mode != FCN_REFINE_MATCHED) return invalid(fn, "labels need FCN_REFINE_MATCHED mode");
    if (a->num_kept == 0) return FCN_OK;
    if (!a->kept || !a->job_data || !a->lists || !a->records || !a->words || (a->labels && !a->job_gt) ||
        (a->labels && a->num_gt > 0 && !a->gt_terms))
        return invalid(fn, "NULL pointer");
    return FCN_OK;
}

}  // namespace fcn

using namespace fcn;

extern "C" int fcn_refine_jobs_from_rows(const fcn_refine_jobs_args *a, fcn_stream_t stream) {
    const int st = rj_check(a, __func__);
    if (st != FCN_OK || a->num_jobs == 0) return st;
    rj_jobs_kernel<<<ceil_div(a->num_jobs, RJ_THREADS), RJ_THREADS, 0, (cudaStream_t)stream>>>(*a);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

extern "C" int fcn_refine_frustum_table(const fcn_refine_frustum_table_args *a, fcn_stream_t stream) {
    const int st = rt_check(a, __func__);
    if (st != FCN_OK || a->num_kept == 0) return st;
    rj_table_kernel<<<ceil_div(a->num_kept, RJ_THREADS), RJ_THREADS, 0, (cudaStream_t)stream>>>(*a);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}
