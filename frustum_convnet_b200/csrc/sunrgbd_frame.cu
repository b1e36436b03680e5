// fcn_sunrgbd_frame_extract (C ABI section (23)): section (18)'s from_rgb_detection set for F frames of fixed
// capacities, every size read on the device and the 2048-point cap drawn there.  Slot f * D + j is detection j of
// frame f.  In order:
//   sf_setup     clamped cloud counts, the status bits and the candidate slots;
//   sf_project   float64 u, v of every cloud point (sx_project_point, the fixed-stride layout read in place);
//   sf_points    <false>: points-major count.  CTA (c, f) takes chunk c of frame f's points and tests each against all
//                of the frame's boxes (in shared memory), one bit per box, and writes per-(slot, chunk) counts;
//   sf_scan      per slot, an exclusive scan over its chunks: n and each chunk's first in-box rank (scan order);
//   sf_slots     one CTA: the n < 5 drop, each frame's P_out budget, the class ranks, the batch entry and output
//                position of every kept frustum, the dummy entries and the cap draw's offsets;
//   resample_choice_kernel (unchanged, through fcn_resample_choice): the cap draw of every slot with n > 2048;
//   sf_sort      each kept capped row's ranks sorted, with the output row of each (choice order);
//   sf_points    <true>: the same traversal writes every kept in-box point at base + rank, or for a capped slot at
//                base + its row in the draw when the rank was drawn;
//   sf_records   one thread per batch entry: its fcn_train_frustum record.
// At F = 1 and P = 393216 the count and write passes run 384 CTAs over the frame where a CTA per slot would run D.
#include <cmath>

#include <cub/block/block_radix_sort.cuh>
#include <cub/block/block_scan.cuh>

#include "common.cuh"
#include "frame_plan.cuh"
#include "input_builder.cuh"
#include "sunrgbd_uv.cuh"

namespace fcn {

constexpr int SF_THREADS = 256;
constexpr int SF_ITEMS = 4;                         // points per thread of a chunk
constexpr int SF_CHUNK = SF_THREADS * SF_ITEMS;
constexpr int SF_WARPS = SF_THREADS / 32;
constexpr int SF_SLOT_THREADS = 1024;
constexpr int SF_CAP = FCN_SUNRGBD_MAX_POINTS;
constexpr int SF_CLASSES = FCN_SUNRGBD_FRAME_CLASSES;
constexpr int SF_MAX_DETS = FCN_SUNRGBD_FRAME_MAX_DETS;
constexpr int SF_MIN_POINTS = 5;                    // prepare_data.py:352
constexpr int SF_SORT_ITEMS = SF_CAP / SF_THREADS;

struct SfWs {
    int32_t *n;                 // (F) clamped cloud counts
    int32_t *ident;             // (B) slot b: the cap draw's key
    int32_t *det_frame;         // (B) f for a candidate slot, else -1
    int32_t *chunk;             // (B, C) per-chunk counts, then each chunk's first in-box rank
    int32_t *det_points;        // (B) n, -1 for a non-candidate
    int32_t *c2, *kept;         // (B) kept points of a slot (-1: dropped); slot of batch entry k (-1: dummy)
    int32_t *cap_off;           // (B + 1) the cap draw's offsets: n for a slot with n > 2048, else 0
    int32_t *ranks, *rows;      // (B, 2048) a capped row's ranks sorted and the draw position of each
    long long *base;            // (B) first output row of a kept slot
    double *u, *v;              // (F * P) image coordinates
    int32_t T[FCN_MAX_SCALES];  // len(np.arange(0, max_depth, stride[s]))
};

// one thread per slot (and per frame for d < F)
__global__ void __launch_bounds__(SF_THREADS) sf_setup_kernel(const fcn_sunrgbd_frame_extract_args a, SfWs w) {
    const int F = a.num_frames, P = a.point_capacity, D = a.det_capacity, B = F * D;
    const int d = blockIdx.x * SF_THREADS + threadIdx.x;
    if (d >= B) return;
    int bits = 0;
    if (d < F) w.n[d] = frame_count(a.cloud_counts[d], a.det_counts[d], P, D, bits);
    w.det_frame[d] = frame_candidate(d, D, SF_CLASSES, a.class_mask, a.det_counts, a.det_class, a.boxes, bits);
    w.ident[d] = d;
    if (bits) atomicOr(a.status, bits);
}

// grid (P / SF_THREADS, F)
__global__ void __launch_bounds__(SF_THREADS) sf_project_kernel(const fcn_sunrgbd_frame_extract_args a, SfWs w) {
    __shared__ double m[18];
    const int f = blockIdx.y, i = blockIdx.x * SF_THREADS + threadIdx.x;
    if (threadIdx.x < 9) m[threadIdx.x] = a.frames[f].Rtilt[threadIdx.x];
    else if (threadIdx.x < 18) m[threadIdx.x] = a.frames[f].K[threadIdx.x - 9];
    __syncthreads();
    if (i >= w.n[f]) return;
    const size_t g = (size_t)f * a.point_capacity + i;
    const float *p = a.clouds + 6 * g;
    sx_project_point(m, m + 9, p[0], p[1], p[2], w.u[g], w.v[g]);
}

// position of rank r in the sorted ranks rk[0, SF_CAP), or -1 when it was not drawn
__device__ __forceinline__ int sf_drawn(const int32_t *__restrict__ rk, int r) {
    int lo = 0, hi = SF_CAP;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (rk[mid] < r) lo = mid + 1;
        else hi = mid;
    }
    return lo < SF_CAP && rk[lo] == r ? lo : -1;
}

// grid (C, F): chunk c of frame f's points, point i = c * SF_CHUNK + q * SF_THREADS + threadIdx.x in round q, so the
// rounds, warps and lanes visit the chunk in scan order.  A point's in-box bits m (bit j: box j of the frame) give,
// per box and round, a warp ballot; the warp counts and the running count run[j] give each in-box point its rank.
// kWrite = false: run[j] ends as the chunk's count of slot j.  kWrite = true: run[j] starts at the chunk's first rank
// and every in-box point of a kept slot is stored.  Four CTAs an SM: without that bound ptxas holds the write pass to
// 32 registers and spills.
template <bool kWrite>
__global__ void __launch_bounds__(SF_THREADS, 4)
sf_points_kernel(const fcn_sunrgbd_frame_extract_args a, SfWs w, int C) {
    __shared__ double box[SF_MAX_DETS][4];
    __shared__ int wcnt[SF_WARPS][SF_MAX_DETS], run[SF_MAX_DETS], kc[SF_MAX_DETS], capped[SF_MAX_DETS];
    __shared__ long long base[SF_MAX_DETS];
    const int f = blockIdx.y, c = blockIdx.x, D = a.det_capacity, n = w.n[f], p0 = c * SF_CHUNK;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int j = threadIdx.x; j < D; j += SF_THREADS) {
        const int d = f * D + j;
        const bool on = p0 < n && (kWrite ? w.c2[d] >= 0 : w.det_frame[d] >= 0);
        for (int q = 0; q < 4; ++q) box[j][q] = on ? a.boxes[4 * (size_t)d + q] : __longlong_as_double(-1ll);  // NaN
        run[j] = kWrite && on ? w.chunk[(size_t)d * C + c] : 0;
        if (kWrite) {
            kc[j] = w.c2[d];
            capped[j] = w.det_points[d] > SF_CAP;
            base[j] = w.base[d];
        }
    }
    __syncthreads();
    for (int q = 0; q < SF_ITEMS && p0 < n; ++q) {
        const int i = p0 + q * SF_THREADS + threadIdx.x;
        const size_t g = (size_t)f * a.point_capacity + i;
        unsigned long long m = 0;
        if (i < n) {
            const double u = w.u[g], v = w.v[g];
            for (int j = 0; j < D; ++j)
                if (sx_in_uv_box(u, v, box[j])) m |= 1ull << j;
        }
        for (int j = 0; j < D; ++j) {
            const unsigned b = __ballot_sync(0xffffffffu, (m >> j) & 1);
            if (lane == 0) wcnt[warp][j] = __popc(b);
        }
        __syncthreads();
        if (kWrite) {
            const unsigned lt = (1u << lane) - 1u;
            for (int j = 0; j < D; ++j) {
                const unsigned b = __ballot_sync(0xffffffffu, (m >> j) & 1);
                if (!((m >> j) & 1)) continue;
                int r = run[j] + __popc(b & lt);
                for (int x = 0; x < warp; ++x) r += wcnt[x][j];
                const int d = f * D + j;
                int o = r;
                if (capped[j]) {
                    const int t = sf_drawn(w.ranks + (size_t)d * SF_CAP, r);
                    o = t >= 0 ? w.rows[(size_t)d * SF_CAP + t] : -1;
                }
                if (o < 0 || o >= kc[j]) continue;
                const float *p = a.clouds + 6 * g;
                const long long t = base[j] + o;
                float *y = a.points + 6 * t;
                y[0] = p[0];
                y[1] = -p[2];
                y[2] = p[1];
                y[3] = p[3];
                y[4] = p[4];
                y[5] = p[5];
                float *z = a.xyz + 3 * t;
                z[0] = p[0];
                z[1] = -p[2];
                z[2] = p[1];
            }
        }
        __syncthreads();
        for (int j = threadIdx.x; j < D; j += SF_THREADS) {
            int s = 0;
            for (int x = 0; x < SF_WARPS; ++x) s += wcnt[x][j];
            run[j] += s;
        }
        __syncthreads();
    }
    if (!kWrite)
        for (int j = threadIdx.x; j < D; j += SF_THREADS) w.chunk[(size_t)(f * D + j) * C + c] = run[j];
}

// one CTA per slot: exclusive scan of its chunk counts in place; n, or -1 for a non-candidate
__global__ void __launch_bounds__(SF_THREADS) sf_scan_kernel(SfWs w, int C) {
    using Scan = cub::BlockScan<int, SF_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    const int d = blockIdx.x;
    int32_t *ch = w.chunk + (size_t)d * C;
    int run = 0;
    for (int c0 = 0; c0 < C; c0 += SF_THREADS) {
        const int c = c0 + threadIdx.x;
        const int v = c < C ? ch[c] : 0;
        int x, total;
        Scan(tmp).ExclusiveSum(v, x, total);
        if (c < C) ch[c] = run + x;
        run += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) w.det_points[d] = w.det_frame[d] >= 0 ? run : -1;
}

// One CTA, after the scan: frame_plan over the F frames of D detection slots, where a candidate with n >= 5 keeps
// min(n, 2048) points; then the cap draw's offsets.
__global__ void __launch_bounds__(SF_SLOT_THREADS) sf_slots_kernel(const fcn_sunrgbd_frame_extract_args a, SfWs w) {
    using Scan = cub::BlockScan<int, SF_SLOT_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    const int B = a.num_frames * a.det_capacity;
    frame_plan<SF_CLASSES, SF_SLOT_THREADS>(
        a.num_frames, a.det_capacity, a.out_capacity, a.det_class, w.c2, w.base, a.seg_class, a.offsets, a.valid,
        a.cls_index, a.seg, a.status,
        [&](int d, int &) {
            const int n = w.det_points[d];
            return n < SF_MIN_POINTS ? -1 : (n < SF_CAP ? n : SF_CAP);
        },
        [&](int k, int d, int c, long long m) {
            a.det_index[k] = d;
            a.rgb_prob[k] = a.det_prob[d];
            for (int i = 0; i < 4; ++i) a.box2d[4 * (size_t)k + i] = (float)a.boxes[4 * (size_t)d + i];
            w.kept[k] = d;
            a.offsets[k + 1] = (int32_t)(m + c);
        },
        [&](int k, int p) {
            for (int i = 0; i < 6; ++i) a.points[6 * (size_t)p + i] = 0.f;
            for (int i = 0; i < 3; ++i) a.xyz[3 * (size_t)p + i] = 0.f;
            a.det_index[k] = -1;
            a.rgb_prob[k] = 0.f;
            const float bx[4] = {0.f, 0.f, 1.f, 1.f};
            for (int i = 0; i < 4; ++i) a.box2d[4 * (size_t)k + i] = bx[i];
            w.kept[k] = -1;
        });
    int run = 0;
    for (int d0 = 0; d0 < B; d0 += SF_SLOT_THREADS) {
        const int d = d0 + threadIdx.x;
        const int n = d < B && w.det_points[d] > SF_CAP ? w.det_points[d] : 0;
        int x, total;
        Scan(tmp).ExclusiveSum(n, x, total);
        if (d < B) w.cap_off[d] = run + x;
        run += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) w.cap_off[B] = run;
}

// one CTA per slot: a kept capped slot's 2048 drawn ranks sorted, with the draw position (output row) of each
__global__ void __launch_bounds__(SF_THREADS) sf_sort_kernel(const fcn_sunrgbd_frame_extract_args a, SfWs w) {
    using Sort = cub::BlockRadixSort<int, SF_THREADS, SF_SORT_ITEMS, int>;
    __shared__ typename Sort::TempStorage tmp;
    const int d = blockIdx.x;
    if (w.c2[d] < 0 || w.det_points[d] <= SF_CAP) return;
    const int32_t *src = a.cap_choice + (size_t)d * SF_CAP;
    int keys[SF_SORT_ITEMS], vals[SF_SORT_ITEMS];
#pragma unroll
    for (int q = 0; q < SF_SORT_ITEMS; ++q) {
        vals[q] = threadIdx.x * SF_SORT_ITEMS + q;
        keys[q] = src[vals[q]];
    }
    Sort(tmp).Sort(keys, vals, 0, 24);
#pragma unroll
    for (int q = 0; q < SF_SORT_ITEMS; ++q) {
        const size_t t = (size_t)d * SF_CAP + threadIdx.x * SF_SORT_ITEMS + q;
        w.ranks[t] = keys[q];
        w.rows[t] = vals[q];
    }
}

// One thread per batch entry: the FCN_TRAIN_SUNRGBD record (labels = 0) of provider_sample_sunrgbd.py's
// from_rgb_detection branch; records were zeroed by the caller.
__global__ void __launch_bounds__(SF_THREADS) sf_records_kernel(const fcn_sunrgbd_frame_extract_args a, SfWs w) {
    const int B = a.num_frames * a.det_capacity, k = blockIdx.x * SF_THREADS + threadIdx.x;
    if (k >= B) return;
    fcn_train_frustum &r = a.records[k];
    const int d = w.kept[k];
    for (int s = 0; s < a.num_scales; ++s) r.T[s] = w.T[s];
    double angle = 0.0;
    if (d < 0) {
        for (int i = 0; i < 9; ++i) r.K[i] = r.Rtilt[i] = (i % 4 == 0) ? 1.0 : 0.0;
    } else {
        const fcn_sunrgbd_frame &fm = a.frames[d / a.det_capacity];
        const double *b = a.boxes + 4 * (size_t)d, *K = fm.K, *R = fm.Rtilt;
        for (int i = 0; i < 9; ++i) {
            r.K[i] = K[i];
            r.Rtilt[i] = R[i];
        }
        // sunrgbd_extract.frustum_angle: the box centre at depth 20, camera (x, y, 20) -> depth (x, 20, -y) ->
        // Rtilt @ . -> upright camera (X, -Z, Y); -atan2 of its z (Y) and x (X)
        const double cx = (b[0] + b[2]) / 2.0, cy = (b[1] + b[3]) / 2.0;
        const double x = __dmul_rn(cx - K[2], 20.0) / K[0];
        const double y = -(__dmul_rn(cy - K[5], 20.0) / K[4]);
        const double X = dot_fma(R[0], x, R[1], 20.0, R[2], y);
        const double Y = dot_fma(R[3], x, R[4], 20.0, R[5], y);
        angle = -atan2(Y, X);
        r.cx = cx;
        r.cy = cy;
        r.rgb_prob = (double)a.det_prob[d];
        r.cls_index = a.det_class[d];
    }
    double sn, cs;
    r.rot = centre_view_angle(angle, &sn, &cs);
    r.cs = cs;
    r.sn = sn;
}

// ------------------------------------------------------------------------------------------------ host side
static int sf_chunks(const fcn_sunrgbd_frame_extract_args *a) { return ceil_div(a->point_capacity, SF_CHUNK); }

static cudaError_t sf_layout(const fcn_sunrgbd_frame_extract_args *a, Carve &c, SfWs &w) {
    const size_t F = (size_t)a->num_frames, B = F * a->det_capacity, FP = F * a->point_capacity;
    w.n = (int32_t *)c.take(F * 4);
    int32_t **b32[] = {&w.ident, &w.det_frame, &w.det_points, &w.c2, &w.kept};
    for (int32_t **q : b32) *q = (int32_t *)c.take(B * 4);
    w.chunk = (int32_t *)c.take(B * sf_chunks(a) * 4);
    w.cap_off = (int32_t *)c.take((B + 1) * 4);
    w.ranks = (int32_t *)c.take(B * SF_CAP * 4);
    w.rows = (int32_t *)c.take(B * SF_CAP * 4);
    w.base = (long long *)c.take(B * 8);
    w.u = (double *)c.take(FP * 8);
    w.v = (double *)c.take(FP * 8);
    return cudaSuccess;
}

// the capacities and the record settings, which alone size the workspace
static int sf_check_sizes(const fcn_sunrgbd_frame_extract_args *a, const char *fn) {
    if (a == nullptr) return invalid(fn, "NULL args");
    const long long F = a->num_frames, P = a->point_capacity, D = a->det_capacity, Po = a->out_capacity;
    if (F < 1 || P < 1 || D < 1 || Po < 1) return invalid(fn, "capacities must be >= 1");
    if (D > SF_MAX_DETS) return invalid(fn, "det_capacity must be <= 64 (one in-box bit per detection of a frame)");
    if (F > 65535 || P >= (1 << 24) || F * P > (1 << 30) || F * D * P >= (1LL << 31) || Po >= (1 << 24) ||
        F * Po + F * D >= (1LL << 31))
        return invalid(fn, "too large (F <= 65535, P < 2^24, F * P <= 2^30, F * D * P < 2^31, P_out < 2^24, "
                           "F * (P_out + D) < 2^31)");
    if (a->class_mask >= (1u << SF_CLASSES)) return invalid(fn, "class_mask has bits past the 10 classes");
    if (a->num_scales < 1 || a->num_scales > FCN_MAX_SCALES) return invalid(fn, "num_scales must be in [1, 8]");
    if (!(a->max_depth > 0.0) || !std::isfinite(a->max_depth)) return invalid(fn, "max_depth must be positive");
    for (int s = 0; s < a->num_scales; ++s)
        if (!(a->stride[s] > 0.0) || !std::isfinite(a->stride[s]) || a->max_depth / a->stride[s] > (1 << 20))
            return invalid(fn, "strides must be positive, with max_depth / stride <= 2^20");
    return FCN_OK;
}

static int sf_check(const fcn_sunrgbd_frame_extract_args *a, const char *fn) {
    const int st = sf_check_sizes(a, fn);
    if (st != FCN_OK) return st;
    if (!a->clouds || !a->cloud_counts || !a->frames || !a->boxes || !a->det_class || !a->det_prob ||
        !a->det_counts || !a->call || !a->status)
        return invalid(fn, "NULL input");
    if (!a->points || !a->xyz || !a->offsets || !a->det_index || !a->valid || !a->cls_index || !a->seg ||
        !a->seg_class || !a->rgb_prob || !a->box2d || !a->cap_choice || !a->records)
        return invalid(fn, "NULL output");
    if (((uintptr_t)a->clouds & 3) != 0) return invalid(fn, "clouds must be 4-byte aligned");
    return FCN_OK;
}

}  // namespace fcn

using namespace fcn;

extern "C" long long fcn_sunrgbd_frame_extract_workspace_bytes(const fcn_sunrgbd_frame_extract_args *a) {
    if (sf_check_sizes(a, __func__) != FCN_OK) return -1;
    SfWs w;
    return workspace_size(__func__, [&](Carve &c) { return sf_layout(a, c, w); });
}

extern "C" int fcn_sunrgbd_frame_extract(const fcn_sunrgbd_frame_extract_args *a, fcn_stream_t stream) {
    int st = sf_check(a, __func__);
    if (st != FCN_OK) return st;
    SfWs w;
    st = carve_workspace(__func__, "sunrgbd_frame_extract", a->workspace, a->workspace_bytes,
                         [&](Carve &c) { return sf_layout(a, c, w); });
    if (st != FCN_OK) return st;
    for (int s = 0; s < FCN_MAX_SCALES; ++s)      // numpy's arange length, ceil((stop - start) / step)
        w.T[s] = s < a->num_scales ? (int32_t)std::ceil(a->max_depth / a->stride[s]) : 0;
    cudaStream_t s = (cudaStream_t)stream;
    const int F = a->num_frames, P = a->point_capacity, B = F * a->det_capacity, C = sf_chunks(a);
    sf_setup_kernel<<<ceil_div(B, SF_THREADS), SF_THREADS, 0, s>>>(*a, w);
    FCN_LAUNCH_CHECK();
    sf_project_kernel<<<dim3(ceil_div(P, SF_THREADS), F), SF_THREADS, 0, s>>>(*a, w);
    FCN_LAUNCH_CHECK();
    sf_points_kernel<false><<<dim3(C, F), SF_THREADS, 0, s>>>(*a, w, C);
    FCN_LAUNCH_CHECK();
    sf_scan_kernel<<<B, SF_THREADS, 0, s>>>(w, C);
    FCN_LAUNCH_CHECK();
    sf_slots_kernel<<<1, SF_SLOT_THREADS, 0, s>>>(*a, w);
    FCN_LAUNCH_CHECK();
    fcn_resample_args r{};
    r.B = B;
    r.N = SF_CAP;
    r.seed = a->seed;
    r.offsets = w.cap_off;
    r.det_index = w.ident;
    r.call = a->call;
    r.choice = a->cap_choice;
    st = fcn_resample_choice(&r, stream);
    if (st != FCN_OK) return st;
    sf_sort_kernel<<<B, SF_THREADS, 0, s>>>(*a, w);
    FCN_LAUNCH_CHECK();
    sf_points_kernel<true><<<dim3(C, F), SF_THREADS, 0, s>>>(*a, w, C);
    FCN_LAUNCH_CHECK();
    FCN_CUDA(cudaMemsetAsync(a->records, 0, (size_t)B * sizeof(fcn_train_frustum), s));
    sf_records_kernel<<<ceil_div(B, SF_THREADS), SF_THREADS, 0, s>>>(*a, w);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}
