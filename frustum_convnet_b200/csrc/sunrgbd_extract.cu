// SUN-RGBD frustums on the device (C ABI section (18)): the point work of extract_frustum_data and
// extract_frustum_data_from_rgb_detection (sunrgbd/prepare_data.py:132-381) for several frames and all their jobs in
// one set of calls.  A job is one cutting 2-D box (and, for the ground-truth sets, one label 3-D box) in one frame.
//
// The reference projects every cloud in numpy, then per box and augmentation cuts the frustum, runs one scipy
// Delaunay for the labels and draws a 2048-point subsample with np.random.choice.  How far that draw advances the
// generator depends on the job's point count, and in the perturbed training set the next box is drawn after it, so
// the host counts before it draws (sunrgbd_extract.py's rounds).  Here:
//   fcn_sunrgbd_extract_project  float64 u, v of every scan point (Rtilt, K; no bounds test, no compaction);
//   fcn_sunrgbd_extract_count    one CTA per job of [job_begin, job_end) over its frame's points: the in-box count n
//                                and the labelled count (box_contains.cuh), read back by the host;
//   fcn_sunrgbd_extract_select   one CTA per job: for a job with n > 2048 the labelled points among the 2048 chosen
//                                (each in-box point's rank from a block scan, binary-searched in the sorted ranks),
//                                the drop rules (prepare_data.py:225-227, :351-353), then the job scans and info;
//   fcn_sunrgbd_extract_write    one CTA per kept job: (x, -z, y, r, g, b) and the labels, in scan order or, for a
//                                capped job, at the output row of each chosen rank (choice order).
#include "box_contains.cuh"
#include "common.cuh"
#include "frustum_fov.cuh"
#include "input_builder.cuh"
#include "sunrgbd_uv.cuh"

namespace fcn {

constexpr int SX_CAP = FCN_SUNRGBD_MAX_POINTS;
constexpr int SX_MIN_POINTS = 5;       // prepare_data.py:226 (labelled points) and :352 (points)

// project_upright_depth_to_image (sunrgbd_utils.py:109-123): d = Rtilt^T p, camera (d0, -d2, d1), (u, v, w) = K cam,
// every np.dot in dgemm's order (dot_fma), then u / w and v / w.
__global__ void __launch_bounds__(FX_THREADS)
sx_project_kernel(const float *__restrict__ scans, const int32_t *__restrict__ so,
                  const fcn_sunrgbd_frame *__restrict__ frames, double *__restrict__ u, double *__restrict__ v) {
    __shared__ double m[18];
    const int f = blockIdx.y;
    if (threadIdx.x < 18) m[threadIdx.x] = frames[f].Rtilt[threadIdx.x];      // Rtilt, K are contiguous
    __syncthreads();
    const int i = so[f] + blockIdx.x * FX_THREADS + threadIdx.x;
    if (i >= so[f + 1]) return;
    const double *R = m, *K = m + 9;
    const double x = scans[6 * (size_t)i], y = scans[6 * (size_t)i + 1], z = scans[6 * (size_t)i + 2];
    const double d0 = dot_fma(R[0], x, R[3], y, R[6], z);
    const double d1 = dot_fma(R[1], x, R[4], y, R[7], z);
    const double d2 = dot_fma(R[2], x, R[5], y, R[8], z);
    const double c0 = d0, c1 = -d2, c2 = d1;
    const double w = dot_fma(c0, K[6], c1, K[7], c2, K[8]);
    u[i] = dot_fma(c0, K[0], c1, K[1], c2, K[2]) / w;
    v[i] = dot_fma(c0, K[3], c1, K[4], c2, K[5]) / w;
}

__device__ __forceinline__ bool sx_in_box2d(double u, double v, const fcn_gt_job &jb) {
    return sx_in_uv_box(u, v, jb.box);
}

// scan point i in upright camera coordinates (x, -z, y), exactly (flip_axis_to_camera)
__device__ __forceinline__ float4 sx_camera(const float *__restrict__ scans, int i) {
    const float *p = scans + 6 * (size_t)i;
    return make_float4(p[0], -p[2], p[1], 0.f);
}

// position of rank r in the sorted ranks rk[0, SX_CAP), or -1 when it was not chosen
__device__ __forceinline__ int sx_chosen(const int32_t *rk, long long r) {
    int lo = 0, hi = SX_CAP;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (rk[mid] < r) lo = mid + 1;
        else hi = mid;
    }
    return lo < SX_CAP && rk[lo] == r ? lo : -1;
}

__device__ __forceinline__ void sx_load_ranks(const int32_t *__restrict__ src, int32_t *rk) {
    for (int t = threadIdx.x; t < SX_CAP; t += FX_THREADS) rk[t] = src[t];
    __syncthreads();
}

template <bool kLabels>
__global__ void __launch_bounds__(FX_THREADS)
sx_count_kernel(int job_begin, int num_frames, int num_labels, const int32_t *__restrict__ so,
                const fcn_gt_job *__restrict__ jobs, const fcn_refine_box *__restrict__ label_boxes,
                const float *__restrict__ scans, const double *__restrict__ u, const double *__restrict__ v,
                int32_t *__restrict__ job_points, int32_t *__restrict__ job_labelled, int32_t *__restrict__ bad) {
    const int j = job_begin + blockIdx.x;
    const fcn_gt_job jb = jobs[j];
    const int f = jb.frame, g = jb.label;
    if (f < 0 || f >= num_frames || (kLabels && (g < 0 || g >= num_labels))) {
        if (threadIdx.x == 0) {
            job_points[j] = -1;
            job_labelled[j] = 0;
            atomicAdd(bad, 1);
        }
        return;
    }
    fcn_refine_box lab;
    if (kLabels) lab = label_boxes[g];
    int c, l;
    job_count<kLabels>(so[f], so[f + 1], c, l, [&](int i, int &c, int &l) {
        if (sx_in_box2d(u[i], v[i], jb)) {
            ++c;
            if (kLabels) l += box3d_contains(lab, sx_camera(scans, i));
        }
    });
    if (threadIdx.x == 0) {
        job_points[j] = c;
        job_labelled[j] = l;
    }
}

template <bool kLabels>
__global__ void __launch_bounds__(FX_THREADS)
sx_select_kernel(int num_choices, const int32_t *__restrict__ so, const fcn_gt_job *__restrict__ jobs,
                 const fcn_refine_box *__restrict__ label_boxes, const float *__restrict__ scans,
                 const double *__restrict__ u, const double *__restrict__ v, int32_t *job_points,
                 const int32_t *__restrict__ job_labelled, const int32_t *__restrict__ job_choice,
                 const int32_t *__restrict__ choice_ranks, int32_t *__restrict__ keep,
                 long long *__restrict__ cnt, int32_t *__restrict__ bad) {
    const int j = blockIdx.x, n = job_points[j], ch = job_choice[j];
    __syncthreads();                           // every thread has read n before thread 0 overwrites it
    if (n < 0 || (n > SX_CAP) != (ch >= 0) || ch >= num_choices) {       // dropped by count, or draws that disagree
        if (threadIdx.x == 0) {
            job_words(j, true, 0, job_points, keep, cnt);
            if (n >= 0) atomicAdd(bad, 1);
        }
        return;
    }
    if (n <= SX_CAP || !kLabels) {
        if (threadIdx.x == 0)
            job_words(j, kLabels ? job_labelled[j] < SX_MIN_POINTS : n < SX_MIN_POINTS, n < SX_CAP ? n : SX_CAP,
                      job_points, keep, cnt);
        return;
    }
    __shared__ int32_t rk[SX_CAP];
    sx_load_ranks(choice_ranks + (size_t)ch * SX_CAP, rk);
    const fcn_gt_job jb = jobs[j];
    const fcn_refine_box lab = label_boxes[jb.label];
    int l = 0;
    job_scatter(so[jb.frame], so[jb.frame + 1], n, 0, [&](int i) { return sx_in_box2d(u[i], v[i], jb); },
                [&](long long r, int i) {
                    if (sx_chosen(rk, r) >= 0) l += box3d_contains(lab, sx_camera(scans, i));
                });
    using Reduce = cub::BlockReduce<int, FX_THREADS>;
    __shared__ typename Reduce::TempStorage tmp;
    l = Reduce(tmp).Sum(l);
    if (threadIdx.x == 0) job_words(j, l < SX_MIN_POINTS, SX_CAP, job_points, keep, cnt);
}

template <bool kLabels>
__global__ void __launch_bounds__(FX_THREADS)
sx_write_kernel(int num_kept, long long num_out, const int32_t *__restrict__ so, const fcn_gt_job *__restrict__ jobs,
                const fcn_refine_box *__restrict__ label_boxes, const float *__restrict__ scans,
                const double *__restrict__ u, const double *__restrict__ v, const int32_t *__restrict__ job_points,
                const int32_t *__restrict__ job_choice,
                const int32_t *__restrict__ choice_ranks, const int32_t *__restrict__ choice_slots,
                const int32_t *__restrict__ keep_pos, const long long *__restrict__ cnt_pos,
                float *__restrict__ points, uint8_t *__restrict__ labels, int32_t *__restrict__ offsets) {
    const int j = blockIdx.x, c = job_points[j];
    int k;
    long long base;
    if (!kept_slot(j, c, num_kept, num_out, keep_pos, cnt_pos, offsets, &k, &base)) return;
    const fcn_gt_job jb = jobs[j];
    fcn_refine_box lab;
    if (kLabels) lab = label_boxes[jb.label];
    auto in = [&](int i) { return sx_in_box2d(u[i], v[i], jb); };
    auto put = [&](long long o, int i) {
        const float *p = scans + 6 * (size_t)i;
        float *q = points + 6 * o;
        q[0] = p[0];
        q[1] = -p[2];
        q[2] = p[1];
        q[3] = p[3];
        q[4] = p[4];
        q[5] = p[5];
        if (kLabels) labels[o] = box3d_contains(lab, sx_camera(scans, i)) ? 1 : 0;
    };
    const int ch = job_choice[j];
    if (ch < 0) {
        job_scatter(so[jb.frame], so[jb.frame + 1], c, base, in, put);
        return;
    }
    __shared__ int32_t rk[SX_CAP];
    sx_load_ranks(choice_ranks + (size_t)ch * SX_CAP, rk);
    const int32_t *slots = choice_slots + (size_t)ch * SX_CAP;
    job_scatter(so[jb.frame], so[jb.frame + 1], INT32_MAX, 0, in, [&](long long r, int i) {
        const int t = sx_chosen(rk, r);
        if (t >= 0) put(base + slots[t], i);
    });
}

// ------------------------------------------------------------------------------------------------ host side
struct SxWs : JobWs {
    double *u, *v;          // image coordinates of every scan point
};

static cudaError_t sx_layout(const fcn_sunrgbd_extract_args *a, Carve &c, SxWs &w) {
    const size_t N = (size_t)a->num_points;
    w.u = (double *)c.take(N * 8);
    w.v = (double *)c.take(N * 8);
    return job_carve(c, a->num_jobs, 0, w);
}

static bool sx_empty(const fcn_sunrgbd_extract_args *a) { return a->num_frames == 0 || a->num_jobs == 0; }

// Host-side checks shared by every entry: counts, pointers, the scan offsets.  Sets *max_n to the largest scan.
static int sx_check(const fcn_sunrgbd_extract_args *a, const char *fn, int *max_n) {
    if (a == nullptr) return invalid(fn, "NULL args");
    if (a->num_frames < 0 || a->num_points < 0 || a->num_jobs < 0 || a->num_labels < 0 || a->num_choices < 0)
        return invalid(fn, "negative count (num_frames, num_points, num_jobs, num_labels, num_choices must be >= 0)");
    if (a->num_frames > 65535 || a->num_points > (1 << 28) || a->num_jobs > (1 << 28) || a->num_labels > (1 << 28) ||
        a->num_choices > a->num_jobs)
        return invalid(fn, "too large (num_frames <= 65535, num_points, num_jobs, num_labels <= 2^28, "
                           "num_choices <= num_jobs)");
    if (a->labelled != 0 && a->labelled != 1) return invalid(fn, "labelled must be 0 or 1");
    *max_n = 0;
    if (sx_empty(a)) return FCN_OK;
    if (!a->scan_offsets || !a->frames || !a->jobs || (a->labelled && !a->label_boxes) ||
        (a->num_points > 0 && !a->scans))
        return invalid(fn, "NULL pointer");
    return check_scans(fn, a->host_scan_offsets, a->num_frames, a->num_points, a->scans, 4, max_n);
}

static int sx_prepare(const fcn_sunrgbd_extract_args *a, const char *fn, SxWs &w, int *max_n) {
    const int st = sx_check(a, fn, max_n);
    if (st != FCN_OK || sx_empty(a)) return st;
    if (!a->workspace || !a->job_points || !a->job_labelled)
        return invalid(fn, "NULL workspace, job_points or job_labelled");
    return carve_workspace(fn, "sunrgbd_extract", a->workspace, a->workspace_bytes,
                           [&](Carve &c) { return sx_layout(a, c, w); });
}

}  // namespace fcn

using namespace fcn;

extern "C" long long fcn_sunrgbd_extract_workspace_bytes(const fcn_sunrgbd_extract_args *a) {
    int max_n;
    if (sx_check(a, __func__, &max_n) != FCN_OK) return -1;
    if (sx_empty(a)) return 0;
    SxWs w;
    return workspace_size(__func__, [&](Carve &c) { return sx_layout(a, c, w); });
}

extern "C" int fcn_sunrgbd_extract_project(const fcn_sunrgbd_extract_args *a, fcn_stream_t stream) {
    SxWs w;
    int max_n;
    const int st = sx_prepare(a, __func__, w, &max_n);
    if (st != FCN_OK || sx_empty(a)) return st;
    cudaStream_t s = (cudaStream_t)stream;
    FCN_CUDA(job_reset(w, a->num_jobs, s));
    if (max_n == 0) return FCN_OK;
    sx_project_kernel<<<dim3(ceil_div(max_n, FX_THREADS), a->num_frames), FX_THREADS, 0, s>>>(
        a->scans, a->scan_offsets, a->frames, w.u, w.v);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

extern "C" int fcn_sunrgbd_extract_count(const fcn_sunrgbd_extract_args *a, fcn_stream_t stream) {
    SxWs w;
    int max_n;
    const int st = sx_prepare(a, __func__, w, &max_n);
    if (st != FCN_OK || sx_empty(a)) return st;
    if (a->job_begin < 0 || a->job_begin > a->job_end || a->job_end > a->num_jobs)
        return invalid(__func__, "need 0 <= job_begin <= job_end <= num_jobs");
    const int n = a->job_end - a->job_begin;
    if (n == 0) return FCN_OK;
    cudaStream_t s = (cudaStream_t)stream;
    if (a->labelled)
        sx_count_kernel<true><<<n, FX_THREADS, 0, s>>>(a->job_begin, a->num_frames, a->num_labels, a->scan_offsets,
                                                       a->jobs, a->label_boxes, a->scans, w.u, w.v, a->job_points,
                                                       a->job_labelled, w.bad);
    else
        sx_count_kernel<false><<<n, FX_THREADS, 0, s>>>(a->job_begin, a->num_frames, a->num_labels, a->scan_offsets,
                                                        a->jobs, nullptr, a->scans, w.u, w.v, a->job_points,
                                                        a->job_labelled, w.bad);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

extern "C" int fcn_sunrgbd_extract_select(const fcn_sunrgbd_extract_args *a, fcn_stream_t stream) {
    SxWs w;
    int max_n;
    const int st = sx_prepare(a, __func__, w, &max_n);
    if (st != FCN_OK || sx_empty(a)) return st;
    if (!a->info || !a->job_choice || (a->num_choices > 0 && !a->choice_ranks))
        return invalid(__func__, "NULL info, job_choice or choice_ranks");
    cudaStream_t s = (cudaStream_t)stream;
    const int J = a->num_jobs;
    if (a->labelled)
        sx_select_kernel<true><<<J, FX_THREADS, 0, s>>>(a->num_choices, a->scan_offsets, a->jobs, a->label_boxes,
                                                        a->scans, w.u, w.v, a->job_points, a->job_labelled,
                                                        a->job_choice, a->choice_ranks, w.keep, w.cnt, w.bad);
    else
        sx_select_kernel<false><<<J, FX_THREADS, 0, s>>>(a->num_choices, a->scan_offsets, a->jobs, nullptr, a->scans,
                                                         w.u, w.v, a->job_points, a->job_labelled, a->job_choice,
                                                         a->choice_ranks, w.keep, w.cnt, w.bad);
    FCN_LAUNCH_CHECK();
    FCN_CUDA(job_totals(w, J, a->info, s));
    return FCN_OK;
}

extern "C" int fcn_sunrgbd_extract_write(const fcn_sunrgbd_extract_args *a, fcn_stream_t stream) {
    SxWs w;
    int max_n;
    const int st = sx_prepare(a, __func__, w, &max_n);
    if (st != FCN_OK || sx_empty(a)) return st;
    if (a->num_kept < 0 || a->num_kept > a->num_jobs || a->num_out_points < 0 || a->num_out_points > INT32_MAX)
        return invalid(__func__, "num_kept must be in [0, num_jobs] and num_out_points in [0, 2^31)");
    if (!a->offsets || !a->job_choice || (a->num_out_points > 0 && (!a->points || (a->labelled && !a->labels))) ||
        (a->num_choices > 0 && (!a->choice_ranks || !a->choice_slots)))
        return invalid(__func__, "NULL output, job_choice or choice arrays");
    cudaStream_t s = (cudaStream_t)stream;
    FCN_CUDA(cudaMemsetAsync(a->offsets, 0, 4, s));
    if (a->num_kept == 0) return FCN_OK;
    if (a->labelled)
        sx_write_kernel<true><<<a->num_jobs, FX_THREADS, 0, s>>>(
            a->num_kept, a->num_out_points, a->scan_offsets, a->jobs, a->label_boxes, a->scans, w.u, w.v,
            a->job_points, a->job_choice, a->choice_ranks, a->choice_slots, w.keep_pos, w.cnt_pos,
            a->points, a->labels, a->offsets);
    else
        sx_write_kernel<false><<<a->num_jobs, FX_THREADS, 0, s>>>(
            a->num_kept, a->num_out_points, a->scan_offsets, a->jobs, nullptr, a->scans, w.u, w.v, a->job_points,
            a->job_choice, a->choice_ranks, a->choice_slots, w.keep_pos, w.cnt_pos, a->points, nullptr,
            a->offsets);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}
