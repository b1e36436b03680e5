// fcn_frame_refine_extract (C ABI section (22)): the refinement frustums of one frame-detection result in fixed
// capacities, every size read on the device.  The kernels of sections (20) and (16) run unchanged over the F * J job
// slots (slot f * J + j is job j of frame f), with these around them:
//   fr_plan   each slot's first-stage row, as section (20)'s gather plan of one-job pieces (rj_jobs_kernel reads it);
//   fr_slots  after the count pass and a table pass over every slot: the W[s] section test, each frame's P2_out
//             budget, the batch entry and output position of every kept frustum (what rx_write_kernel is handed), the
//             batch tables and the dummy entries (frame_plan).
// The in-image points are recomputed from the scans (frame_setup, frame_pack and fov_stage of section (21)) rather
// than kept from the detection call: that costs one more pass over the F * P scan points (a flag, a scan and a
// compaction) and saves keeping F * P float4 points and their scan alive between the two calls.
#include <cmath>

#include "common.cuh"
#include "frame_extract.cuh"
#include "frame_plan.cuh"
#include "frame_refine.cuh"
#include "frustum_fov.cuh"

namespace fcn {

constexpr int FR_THREADS = 256;
constexpr int FR_SLOT_THREADS = 1024;

struct FrPlan {
    int32_t *offsets, *row, *frame, *image, *cls;     // one piece per slot (section (20))
};

// One thread per slot d = f * J + j: frame f's jobs are the kept rows of its whitelisted segments 3 f + r, r in
// order, then rows in order.  A slot without a row gets frame -1 (the count pass drops it) and row 0 (read, unused).
__global__ void __launch_bounds__(FR_THREADS) fr_plan_kernel(const fcn_frame_refine_args a, FrPlan p) {
    const int J = a.job_capacity, B = a.num_frames * J, d = blockIdx.x * FR_THREADS + threadIdx.x;
    if (d >= B) return;
    const int f = d / J, j = d - f * J;
    int row = -1, cls = 0, total = 0;
    for (int r = 0; r < 3; ++r) {
        const int c = a.seg_class[3 * f + r];
        if (c < 0 || c > 2 || !((a.class_mask >> c) & 1u)) continue;
        const int n = max(a.keep_count[3 * f + r], 0);
        if (row < 0 && j < total + n) {
            row = a.seg_offsets[3 * f + r] + (j - total);
            cls = c;
        }
        total += n;
    }
    const bool ok = row >= 0 && row < a.num_rows;
    p.offsets[d] = d;
    if (d == B - 1) p.offsets[B] = B;
    p.row[d] = ok ? row : 0;
    p.frame[d] = ok ? f : -1;
    p.image[d] = f;
    p.cls[d] = cls;
    if (j == 0 && total > J) atomicOr(a.status, FCN_FRAME_JOBS);
}

// One CTA, after the count pass and the table pass over every slot (words: T per scale of each slot's record):
// frame_plan over the F frames of J job slots, where a counted frustum whose T[s] exceeds widths[s] is dropped.  The
// dummy entries' record is the one-section box of job_data[B].
__global__ void __launch_bounds__(FR_SLOT_THREADS)
fr_slots_kernel(const fcn_frame_refine_args a, FrPlan p, const int32_t *__restrict__ job_status,
                const int32_t *__restrict__ job_points, const int32_t *__restrict__ words,
                fcn_refine_job_data *__restrict__ job_data, int32_t *__restrict__ c2, int32_t *__restrict__ kpos,
                long long *__restrict__ base, int32_t *__restrict__ kept) {
    const int B = a.num_frames * a.job_capacity, S = a.num_scales;
    frame_plan<3, FR_SLOT_THREADS>(
        a.num_frames, a.job_capacity, a.out_capacity, p.cls, c2, base, a.seg_class_out, a.offsets, a.valid,
        a.cls_index, a.seg, a.status,
        [&](int d, int &bits) {
            if (p.frame[d] >= 0 && (job_status[d] & (FCN_REFINE_ROW_NONFINITE | FCN_REFINE_ROW_EXTENTS)))
                bits |= FCN_FRAME_BAD_DET;
            if (job_points[d] < 0) return -1;
            bool fits = true;
            for (int s = 0; s < S; ++s) fits = fits && words[(size_t)d * (S + 1) + s] <= a.widths[s];
            if (!fits) bits |= FCN_FRAME_SECTIONS;
            return fits ? job_points[d] : -1;
        },
        [&](int k, int d, int, long long) {
            kpos[d] = k;
            a.job_index[k] = d;
            kept[k] = d;
            for (int i = 0; i < 4; ++i) a.box2d[4 * (size_t)k + i] = (float)job_data[d].box2d[i];
        },
        [&](int k, int pt) {
            reinterpret_cast<float4 *>(a.points)[pt] = make_float4(0.f, 0.f, 0.f, 0.f);
            a.job_index[k] = -1;
            kept[k] = B;
            const float bx[4] = {0.f, 0.f, 1.f, 1.f};
            for (int i = 0; i < 4; ++i) a.box2d[4 * (size_t)k + i] = bx[i];
        });
    if (threadIdx.x == 0) {
        double w = a.stride[0];                     // T[s] = ceil(w / stride[s]) = 1 at every scale
        for (int s = 1; s < S; ++s) w = fmin(w, a.stride[s]);
        fcn_refine_job_data dd;
        for (int i = 0; i < 7; ++i) dd.cut[i] = (i >= 3 && i < 6) ? w : 0.0;
        const double bx[4] = {0.0, 0.0, 1.0, 1.0};
        for (int i = 0; i < 4; ++i) dd.box2d[i] = bx[i];
        dd.prob = 0.0;
        dd.image = 0;
        dd.cls_index = 0;
        job_data[B] = dd;
    }
}

// ------------------------------------------------------------------------------------------------ host side
struct FrWs : FovWs {
    float4 *packed;
    int32_t *so, *det_frame, *no_dets;
    FrPlan plan;
    fcn_refine_box *jobs;
    int32_t *job_frame, *job_ref, *job_status, *job_points, *job_gt, *c2, *kpos, *kept, *words;
    fcn_refine_job_data *job_data;
    long long *base;
    double *lists;
};

static cudaError_t fr_layout(const fcn_frame_refine_args *a, Carve &c, FrWs &w) {
    const size_t F = (size_t)a->num_frames, FP = F * a->scan_capacity, B = F * a->job_capacity;
    const cudaError_t e = fov_carve(c, (int)FP, (int)B, false, w);
    w.packed = (float4 *)c.take(FP * 16);
    w.so = (int32_t *)c.take((F + 1) * 4);
    w.det_frame = (int32_t *)c.take(F * 4);
    w.no_dets = (int32_t *)c.take(F * 4);
    w.plan.offsets = (int32_t *)c.take((B + 1) * 4);
    int32_t **i32[] = {&w.plan.row, &w.plan.frame, &w.plan.image, &w.plan.cls, &w.job_frame, &w.job_ref,
                       &w.job_status, &w.job_points, &w.job_gt, &w.c2, &w.kpos, &w.kept};
    for (int32_t **q : i32) *q = (int32_t *)c.take(B * 4);
    w.jobs = (fcn_refine_box *)c.take(B * sizeof(fcn_refine_box));
    w.job_data = (fcn_refine_job_data *)c.take((B + 1) * sizeof(fcn_refine_job_data));
    w.base = (long long *)c.take(B * 8);
    w.lists = (double *)c.take(B * FCN_REFINE_LIST_COLS * 8);
    w.words = (int32_t *)c.take(B * (a->num_scales + 1) * 4);
    return e;
}

// the capacities and scales, which alone size the workspace
static int fr_check_sizes(const fcn_frame_refine_args *a, const char *fn) {
    if (a == nullptr) return invalid(fn, "NULL args");
    const long long F = a->num_frames, P = a->scan_capacity, J = a->job_capacity, Po = a->out_capacity;
    if (F < 1 || P < 1 || J < 1 || Po < 1 || a->num_rows < 1) return invalid(fn, "capacities must be >= 1");
    if (F > 65535 || F * P > (1 << 30) || F * J > (1 << 28) || Po >= (1 << 24) || F * Po + F * J >= (1LL << 31))
        return invalid(fn, "too large (F <= 65535, F * P <= 2^30, F * J <= 2^28, P2_out < 2^24, "
                           "F * (P2_out + J) < 2^31)");
    if (a->num_scales < 1 || a->num_scales > FCN_MAX_SCALES) return invalid(fn, "num_scales must be in [1, 8]");
    for (int s = 0; s < a->num_scales; ++s) {
        if (!(a->stride[s] > 0.0) || !std::isfinite(a->stride[s])) return invalid(fn, "strides must be positive");
        if (a->widths[s] < 1) return invalid(fn, "widths must be >= 1");
    }
    return FCN_OK;
}

static int fr_check(const fcn_frame_refine_args *a, const char *fn) {
    const int st = fr_check_sizes(a, fn);
    if (st != FCN_OK) return st;
    if (!a->scans || !a->scan_counts || !a->frames || !a->rows || !a->seg_offsets || !a->keep_count ||
        !a->seg_class || !a->status)
        return invalid(fn, "NULL input");
    if (!a->points || !a->offsets || !a->job_index || !a->valid || !a->cls_index || !a->seg || !a->seg_class_out ||
        !a->records || !a->box2d)
        return invalid(fn, "NULL output");
    if (((uintptr_t)a->scans & 15) != 0 || ((uintptr_t)a->points & 15) != 0)
        return invalid(fn, "scans and points must be 16-byte aligned");
    return FCN_OK;
}

}  // namespace fcn

using namespace fcn;

extern "C" long long fcn_frame_refine_extract_workspace_bytes(const fcn_frame_refine_args *a) {
    if (fr_check_sizes(a, __func__) != FCN_OK) return -1;
    FrWs w;
    return workspace_size(__func__, [&](Carve &c) { return fr_layout(a, c, w); });
}

extern "C" int fcn_frame_refine_extract(const fcn_frame_refine_args *a, fcn_stream_t stream) {
    int st = fr_check(a, __func__);
    if (st != FCN_OK) return st;
    FrWs w;
    st = carve_workspace(__func__, "frame_refine_extract", a->workspace, a->workspace_bytes,
                         [&](Carve &c) { return fr_layout(a, c, w); });
    if (st != FCN_OK) return st;
    cudaStream_t s = (cudaStream_t)stream;
    const int F = a->num_frames, P = a->scan_capacity, B = F * a->job_capacity, S = a->num_scales;
    // jobs: the plan, then section (20)'s job kernel in FCN_REFINE_DET mode
    fr_plan_kernel<<<ceil_div(B, FR_THREADS), FR_THREADS, 0, s>>>(*a, w.plan);
    FCN_LAUNCH_CHECK();
    fcn_refine_jobs_args ja{};
    ja.mode = FCN_REFINE_DET;
    ja.num_pieces = ja.num_jobs = B;
    ja.num_rows = a->num_rows;
    ja.rows = a->rows;
    ja.piece_offsets = w.plan.offsets;
    ja.piece_row = w.plan.row;
    ja.piece_frame = w.plan.frame;
    ja.piece_image = w.plan.image;
    ja.piece_class = w.plan.cls;
    ja.jobs = w.jobs;
    ja.job_frame = w.job_frame;
    ja.job_ref = w.job_ref;
    ja.status = w.job_status;
    ja.job_data = w.job_data;
    FCN_CUDA(rj_jobs(ja, s));
    // points: section (21)'s packed scans and in-image stage (no detection slots), section (16)'s count pass
    fcn_frame_extract_args fx{};
    fx.num_frames = F;
    fx.scan_capacity = P;
    fx.det_capacity = 1;
    fx.scans = a->scans;
    fx.scan_counts = a->scan_counts;
    fx.det_counts = w.no_dets;
    fx.status = a->status;
    FCN_CUDA(cudaMemsetAsync(w.no_dets, 0, (size_t)F * 4, s));
    FCN_CUDA(frame_setup(fx, w.so, w.det_frame, w.packed, s));
    FCN_CUDA(fov_stage(w, F * P, B, F, P, w.packed, w.so, a->frames, s));
    FCN_CUDA(rx_count_det(F, B, w.so, w.jobs, w.job_frame, w.pos, w.fov_pts, w.job_points, w.job_gt, w.keep, w.cnt,
                          w.bad, s));
    // the sections of every slot's record (section (20)'s table, kept = the identity), then the slots
    fcn_refine_frustum_table_args ta{};
    ta.mode = FCN_REFINE_DET;
    ta.num_kept = B;
    ta.num_jobs = B + 1;
    ta.num_scales = S;
    for (int q = 0; q < S; ++q) ta.stride[q] = a->stride[q];
    ta.kept = w.plan.offsets;
    ta.job_data = w.job_data;
    ta.lists = w.lists;
    ta.records = a->records;
    ta.words = w.words;
    FCN_CUDA(rj_table(ta, s));
    fr_slots_kernel<<<1, FR_SLOT_THREADS, 0, s>>>(*a, w.plan, w.job_status, w.job_points, w.words, w.job_data, w.c2,
                                                  w.kpos, w.base, w.kept);
    FCN_LAUNCH_CHECK();
    FCN_CUDA(rx_write_det(B, B, (long long)F * a->out_capacity, w.so, w.jobs, w.job_frame, w.c2, w.job_gt, w.kpos,
                          w.base, w.pos, w.fov_pts, (float4 *)a->points, a->offsets, s));
    // the batch entries' records: the kept frustums' and the dummies' (job_data[B])
    FCN_CUDA(cudaMemsetAsync(a->records, 0, (size_t)B * sizeof(fcn_train_frustum), s));
    ta.kept = w.kept;
    FCN_CUDA(rj_table(ta, s));
    return FCN_OK;
}
