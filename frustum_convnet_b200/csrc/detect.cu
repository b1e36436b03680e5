// Per-image 3-D detections on the device (C ABI section (10)): replaces the host loop of
// train/test_net_det.py:243-293 (test_net_det_sunrgbd.py:197-252) and write_detection_results_nms (:126-152).
//
// fcn_det_candidates, once per batch: one CTA per frustum selects the foreground positions, scores and decodes
// them (from_prediction_to_label_format, provider_sample.py:375-387 / provider_sample_sunrgbd.py:374-385), drops
// tiny boxes and appends one record per row behind a device row counter (one atomicAdd per frustum).
//
// Finalize, once per pass:
//   fcn_det_prepare  1. radix sort of the records by (segment, frustum, t): the reference's list order;
//                    2. rows per segment -> seg_offsets; for 'nms' the bit-matrix words and 32 x 32 pair tiles per
//                       segment (exclusive scans), and a second stable radix sort by (segment, score): read backwards
//                       it is the rank order, descending score with ties larger list index first;
//   (the host reads info = {rows, mask words, tiles} once and allocates the bit matrix)
//   fcn_det_select   3. corners / bounding cubes in rank order; suppression bits of every pair tile of every segment,
//                       the tiles spread over the whole grid (one warp per tile); the pair test is the one of
//                       nms3d.cu (cubes overlap, then rbbox_iou_pair >= thresh);
//                    4. greedy scan, one warp per segment, stops at top_k kept rows;
//                    5. kept rows gathered in keep order into the label-format row layout.
#include <cub/cub.cuh>

#include "box_corners.cuh"
#include "box_iou.cuh"
#include "common.cuh"

namespace fcn {

constexpr int DET_THREADS = 128;
constexpr int DET_ROW = 12;
constexpr int DET_FIN_THREADS = 256;
constexpr unsigned long long DET_KEY_NONE = ~0ull;

static_assert(sizeof(fcn_det_record) == 48, "fcn_det_record is 48 bytes");

// np.argmax order: the first NaN wins, else the largest value, ties -> smaller index
__device__ __forceinline__ bool arg_better(float v, int i, float bv, int bi) {
    if (bi < 0) return i >= 0;
    const bool nv = isnan(v), nb = isnan(bv);
    if (nb) return nv && i < bi;
    if (nv) return true;
    return v > bv || (v == bv && i < bi);
}

__device__ __forceinline__ bool det_is_fg(int dataset, float p0, float p1) {
    return dataset == FCN_DET_KITTI ? (p0 < p1) : (p1 > 0.5f);
}

// h, w or l below 0.01 is dropped (test_net_det.py:290); the fp32 value is compared with 0.01f as numpy >= 2
// compares a float32 scalar with a Python float
__device__ __forceinline__ bool det_size_ok(const float *sz) {
    return !(sz[2] < 0.01f || sz[1] < 0.01f || sz[0] < 0.01f);
}

__global__ void __launch_bounds__(DET_THREADS) det_candidates_kernel(const fcn_det_candidate_args a) {
    __shared__ float s_bv[DET_THREADS / 32];
    __shared__ int s_bi[DET_THREADS / 32], s_n[DET_THREADS / 32], s_base;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, T2 = a.T2;
    const float *p = a.cls_probs + (size_t)b * T2 * 2;
    // ---- foreground count and first argmax of p[:, 1]
    int nfg = 0, bi = -1;
    float bv = 0.f;
    for (int t = tid; t < T2; t += DET_THREADS) {
        const float p0 = p[2 * t], p1 = p[2 * t + 1];
        nfg += det_is_fg(a.dataset, p0, p1) ? 1 : 0;
        if (arg_better(p1, t, bv, bi)) { bv = p1; bi = t; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        nfg += __shfl_xor_sync(0xffffffffu, nfg, o);
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (arg_better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { s_bv[warp] = bv; s_bi[warp] = bi; s_n[warp] = nfg; }
    __syncthreads();
    nfg = 0; bv = 0.f; bi = -1;
    for (int w = 0; w < DET_THREADS / 32; ++w) {
        nfg += s_n[w];
        if (arg_better(s_bv[w], s_bi[w], bv, bi)) { bv = s_bv[w]; bi = s_bi[w]; }
    }
    const bool single = a.method != FCN_DET_NMS || nfg == 0;   // 'top', or the fallback of an all-background frustum
    const float *sz = a.size + (size_t)b * T2 * 3;
    // ---- rows of this thread (positions t = tid, tid + 128, ...), block exclusive scan, one reservation
    int mine = 0;
    for (int t = tid; t < T2; t += DET_THREADS) {
        const bool cand = single ? t == bi : det_is_fg(a.dataset, p[2 * t], p[2 * t + 1]);
        mine += (cand && det_size_ok(sz + 3 * t)) ? 1 : 0;
    }
    int incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    __syncthreads();                                     // s_n is reused
    if (lane == 31) s_n[warp] = incl;
    __syncthreads();
    int excl = incl - mine, total = 0;
    for (int w = 0; w < DET_THREADS / 32; ++w) {
        if (w < warp) excl += s_n[w];
        total += s_n[w];
    }
    if (tid == 0) s_base = total > 0 ? atomicAdd(a.counter, total) : 0;
    __syncthreads();
    if (mine == 0) return;
    // ---- decode and write
    const float r = a.rot_angle[b];
    const float rgb = a.rgb_prob ? a.rgb_prob[b] : 1.f;
    const float r0 = a.ref_center ? a.ref_center[3 * b + 0] : 0.f;
    const float r1 = a.ref_center ? a.ref_center[3 * b + 1] : 0.f;
    const float r2 = a.ref_center ? a.ref_center[3 * b + 2] : 0.f;
    // rotate_pc_along_y(center, -rot_angle): [x, z] <- [x, z] . [[c, -s], [s, c]]^T with c, s of -rot_angle
    const float c = cosf(-r), s = sinf(-r);
    const int frustum = a.first + b;
    const int seg = a.seg_of_frustum[frustum];
    int row = s_base + excl;
    for (int t = tid; t < T2; t += DET_THREADS) {
        const bool cand = single ? t == bi : det_is_fg(a.dataset, p[2 * t], p[2 * t + 1]);
        if (!cand || !det_size_ok(sz + 3 * t)) continue;
        if (row < a.capacity) {
            const size_t bt = (size_t)b * T2 + t;
            const float x = a.center[3 * bt + 0], y = a.center[3 * bt + 1], z = a.center[3 * bt + 2];
            const float l = sz[3 * t + 0], w = sz[3 * t + 1], h = sz[3 * t + 2];
            float score;
            if (a.dataset == FCN_DET_KITTI) {
                score = __fadd_rn(p[2 * t + 1], rgb);
            } else {
                const float *sp = a.size_probs + bt * a.NS;
                float m = sp[0];
                for (int k = 1; k < a.NS; ++k) m = (sp[k] > m || isnan(sp[k])) && !isnan(m) ? sp[k] : m;
                score = __fadd_rn(rgb, m);
            }
            float tx = __fadd_rn(__fmul_rn(x, c), __fmul_rn(z, -s));
            float tz = __fadd_rn(__fmul_rn(x, s), __fmul_rn(z, c));
            tx = __fadd_rn(tx, r0);
            float ty = __fadd_rn(y, r1);
            tz = __fadd_rn(tz, r2);
            if (a.dataset == FCN_DET_KITTI) ty = __fadd_rn(ty, __fmul_rn(h, 0.5f));
            fcn_det_record rec;
            rec.seg = seg;
            rec.frustum = frustum;
            rec.t = t;
            rec.reserved = 0;
            rec.box[0] = tx; rec.box[1] = ty; rec.box[2] = tz;
            rec.box[3] = l; rec.box[4] = w; rec.box[5] = h;
            rec.box[6] = __fadd_rn(a.heading[bt], r);
            rec.box[7] = score;
            a.records[row] = rec;
        }
        ++row;
    }
}

// ---------------------------------------------------------------------------------------------- finalize
// order-preserving map of an fp32 score to uint32 (ascending); -0 is read as +0 so that equal scores tie
__device__ __forceinline__ unsigned score_key(float s) {
    if (s == 0.f) s = 0.f;
    const unsigned u = __float_as_uint(s);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void det_keys_kernel(int capacity, const int32_t *counter, const fcn_det_record *rec,
                                unsigned long long *keys, int *vals, int *seg_cnt) {
    const int n = min(*counter, capacity);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < capacity; i += gridDim.x * blockDim.x) {
        vals[i] = i;
        if (i < n) {
            const fcn_det_record &r = rec[i];
            keys[i] = ((unsigned long long)r.seg << 44) | ((unsigned long long)r.frustum << 16) | (unsigned)r.t;
            atomicAdd(&seg_cnt[r.seg], 1);
        } else {
            keys[i] = DET_KEY_NONE;
        }
    }
}

// sorted records + (nms) the keys of the rank sort: (segment, score) ascending, stable
__global__ void det_gather_sorted_kernel(int capacity, const int32_t *counter, int nms, const fcn_det_record *rec,
                                         const int *order, fcn_det_record *sorted, unsigned long long *keys2,
                                         int *vals2) {
    const int n = min(*counter, capacity);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < capacity; i += gridDim.x * blockDim.x) {
        if (i < n) sorted[i] = rec[order[i]];
        if (nms) {
            vals2[i] = i;
            keys2[i] = i < n ? ((unsigned long long)sorted[i].seg << 32) | score_key(sorted[i].box[7]) : DET_KEY_NONE;
        }
    }
}

// per segment: bit-matrix words n*W and upper-triangle 32 x 32 tiles W(W+1)/2 (lists of >= 2 rows under 'nms')
__global__ void det_seg_sizes_kernel(int S, int nms, const int *seg_cnt, long long *mask_w, long long *tiles) {
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s <= S; s += gridDim.x * blockDim.x) {
        const long long n = s < S ? seg_cnt[s] : 0, W = (n + 31) / 32;
        const bool on = nms && n >= 2;
        mask_w[s] = on ? n * W : 0;
        tiles[s] = on ? W * (W + 1) / 2 : 0;
    }
}

__global__ void det_info_kernel(int S, const int32_t *counter, const long long *mask_off, const long long *tile_off,
                                long long *info) {
    info[0] = *counter;
    info[1] = mask_off[S];
    info[2] = tile_off[S];
    info[3] = 0;
}

// rank g of the whole rank-ordered array (segment s occupies [off[s], off[s+1]) in both orders): the rank sort
// read backwards; corners and bounding cube of that box
__global__ void det_rank_kernel(int n, const fcn_det_record *sorted, const int *seg_off, const int *vals2,
                                int *rank_idx, float *corners, float *cube) {
    for (int g = blockIdx.x * blockDim.x + threadIdx.x; g < n; g += gridDim.x * blockDim.x) {
        const int s = sorted[g].seg;
        const int src = vals2[seg_off[s] + seg_off[s + 1] - 1 - g];
        rank_idx[g] = src;
        float c[24];
        box_to_corners(sorted[src].box, c);
        float mn[3] = {c[0], c[1], c[2]}, mx[3] = {c[0], c[1], c[2]};
#pragma unroll
        for (int i = 0; i < 8; ++i) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                corners[(size_t)g * 24 + 3 * i + k] = c[3 * i + k];
                mn[k] = fminf(mn[k], c[3 * i + k]);
                mx[k] = fmaxf(mx[k], c[3 * i + k]);
            }
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) { cube[(size_t)g * 6 + k] = mn[k]; cube[(size_t)g * 6 + 3 + k] = mx[k]; }
    }
}

// one warp per 32 x 32 tile (row block rb, column word cb >= rb) of one segment's bit matrix, tiles of all
// segments spread over the grid; lane = row.  Words left of the diagonal block are never written nor read.
__global__ void __launch_bounds__(DET_FIN_THREADS)
det_pairs_kernel(int S, float thresh, const int *seg_off, const long long *mask_off, const long long *tile_off,
                 const float *__restrict__ corners, const float *__restrict__ cube, unsigned *__restrict__ mask) {
    const int lane = threadIdx.x & 31;
    const long long total = tile_off[S];
    const long long nwarps = (long long)gridDim.x * (DET_FIN_THREADS / 32);
    for (long long tile = (long long)blockIdx.x * (DET_FIN_THREADS / 32) + (threadIdx.x >> 5); tile < total;
         tile += nwarps) {
        int lo = 0, hi = S;                       // last s with tile_off[s] <= tile
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (tile_off[mid] <= tile) lo = mid; else hi = mid;
        }
        const int s = lo, base = seg_off[s], n = seg_off[s + 1] - base, W = (n + 31) >> 5;
        int rem = (int)(tile - tile_off[s]), rb = 0;
        while (rem >= W - rb) { rem -= W - rb; ++rb; }
        const int cb = rb + rem;
        const int i = rb * 32 + lane;
        if (i >= n) continue;
        const float *ci = corners + (size_t)(base + i) * 24, *ki = cube + (size_t)(base + i) * 6;
        unsigned word = 0u;
        const int j_end = min(n, cb * 32 + 32);
        for (int j = max(cb * 32, i + 1); j < j_end; ++j) {
            if (!cubes_overlap(ki, cube + (size_t)(base + j) * 6)) continue;
            float iou[2];
            rbbox_iou_pair(ci, corners + (size_t)(base + j) * 24, iou);
            if (iou[1] >= thresh) word |= 1u << (j & 31);
        }
        mask[mask_off[s] + (long long)i * W + cb] = word;
    }
}

// greedy scan in rank order, one warp per segment.  removed[] (zeroed) holds the suppressed set, word w owned by
// lane w % 32; the current 32-row word is kept in a register by every lane.  keep[off + k] = rank-space index.
__global__ void __launch_bounds__(DET_FIN_THREADS)
det_scan_kernel(int S, int nms, int top_k, const int *seg_off, const long long *mask_off, const unsigned *mask,
                unsigned *removed, int *keep, int32_t *keep_count) {
    const int lane = threadIdx.x & 31;
    const int nwarps = gridDim.x * (DET_FIN_THREADS / 32);
    for (int s = blockIdx.x * (DET_FIN_THREADS / 32) + (threadIdx.x >> 5); s < S; s += nwarps) {
        const int base = seg_off[s], n = seg_off[s + 1] - base, W = (n + 31) >> 5;
        if (!nms) {
            if (lane == 0) keep_count[s] = n;
            continue;
        }
        unsigned *rm = removed + (base >> 5) + s;
        const unsigned *m = mask + (n >= 2 ? mask_off[s] : 0);
        int kept = 0;
        for (int c = 0; c < W && kept < top_k; ++c) {
            __syncwarp();
            unsigned word = rm[c];
            for (int k = 0; k < 32 && kept < top_k; ++k) {
                const int i = c * 32 + k;
                if (i >= n) break;
                if ((word >> k) & 1u) continue;
                if (lane == 0) keep[base + kept] = base + i;
                ++kept;
                if (n < 2) break;
                const unsigned *row = m + (size_t)i * W;
                word |= row[c];
                for (int w = c + 1 + ((lane - c - 1) & 31); w < W; w += 32) rm[w] |= row[w];
            }
        }
        if (lane == 0) keep_count[s] = kept;
    }
}

__global__ void det_rows_kernel(int n, int nms, int dataset, const fcn_det_record *sorted, const int *seg_off,
                                const int *rank_idx, const int *keep, const int32_t *keep_count, const float *box2d,
                                float *rows) {
    for (int g = blockIdx.x * blockDim.x + threadIdx.x; g < n; g += gridDim.x * blockDim.x) {
        const int s = sorted[g].seg;
        if (g - seg_off[s] >= keep_count[s]) continue;
        const fcn_det_record &r = sorted[nms ? rank_idx[keep[g]] : g];
        float *o = rows + (size_t)g * DET_ROW;
        const float *bx = box2d + (size_t)r.frustum * 4;
        o[0] = bx[0]; o[1] = bx[1]; o[2] = bx[2]; o[3] = bx[3];
        o[4] = r.box[0]; o[5] = r.box[1]; o[6] = r.box[2];
        if (dataset == FCN_DET_KITTI) { o[7] = r.box[5]; o[8] = r.box[4]; o[9] = r.box[3]; }   // h, w, l
        else { o[7] = r.box[3]; o[8] = r.box[4]; o[9] = r.box[5]; }                            // l, w, h
        o[10] = r.box[6];
        o[11] = r.box[7];
    }
}

// ---------------------------------------------------------------------------------------------- workspace
struct DetWs {
    unsigned long long *keys_a, *keys_b;
    int *vals_a, *vals_b, *seg_cnt, *rank_idx, *keep;
    fcn_det_record *sorted;
    long long *mask_w, *tiles, *mask_off, *tile_off;
    float *corners, *cube;
    unsigned *removed;
    void *temp;
    size_t temp_bytes;
};

// returns a CUDA error of the cub size queries
static cudaError_t det_layout(int capacity, int S, Carve &c, DetWs &w) {
    const size_t C = (size_t)capacity;
    size_t t_sort = 0, t_scan32 = 0, t_scan64 = 0;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, t_sort, (unsigned long long *)nullptr,
                                                    (unsigned long long *)nullptr, (int *)nullptr, (int *)nullptr,
                                                    capacity);
    if (e != cudaSuccess) return e;
    e = cub::DeviceScan::ExclusiveSum(nullptr, t_scan32, (int *)nullptr, (int *)nullptr, S + 1);
    if (e != cudaSuccess) return e;
    e = cub::DeviceScan::ExclusiveSum(nullptr, t_scan64, (long long *)nullptr, (long long *)nullptr, S + 1);
    if (e != cudaSuccess) return e;
    w.temp_bytes = std::max(t_sort, std::max(t_scan32, t_scan64));
    w.keys_a = (unsigned long long *)c.take(C * 8);
    w.keys_b = (unsigned long long *)c.take(C * 8);
    w.vals_a = (int *)c.take(C * 4);
    w.vals_b = (int *)c.take(C * 4);
    w.sorted = (fcn_det_record *)c.take(C * sizeof(fcn_det_record));
    w.seg_cnt = (int *)c.take((size_t)(S + 1) * 4);
    w.mask_w = (long long *)c.take((size_t)(S + 1) * 8);
    w.tiles = (long long *)c.take((size_t)(S + 1) * 8);
    w.mask_off = (long long *)c.take((size_t)(S + 1) * 8);
    w.tile_off = (long long *)c.take((size_t)(S + 1) * 8);
    w.rank_idx = (int *)c.take(C * 4);
    w.keep = (int *)c.take(C * 4);
    w.corners = (float *)c.take(C * 24 * 4);
    w.cube = (float *)c.take(C * 6 * 4);
    w.removed = (unsigned *)c.take((C / 32 + (size_t)S + 2) * 4);
    w.temp = c.take(w.temp_bytes);
    return cudaSuccess;
}

static int det_grid(long long work, int threads) {
    return (int)std::max(1LL, std::min((work + threads - 1) / threads, (long long)sm_count() * 8));
}

}  // namespace fcn

using namespace fcn;

extern "C" int fcn_det_candidates(const fcn_det_candidate_args *a, fcn_stream_t stream) {
    FCN_REQUIRE(a != nullptr, "NULL args");
    FCN_REQUIRE(a->B >= 0 && a->T2 >= 1 && a->T2 < 65536 && a->capacity >= 0, "bad sizes (1 <= T2 < 65536)");
    FCN_REQUIRE(a->dataset == FCN_DET_KITTI || a->dataset == FCN_DET_SUNRGBD, "dataset must be 0 (KITTI) or 1 (SUN-RGBD)");
    FCN_REQUIRE(a->method == FCN_DET_NMS || a->method == FCN_DET_TOP, "method must be 0 (nms) or 1 (top)");
    FCN_REQUIRE(a->num_frustums >= 0 && a->num_frustums < (1 << 28), "num_frustums must be < 2^28");
    FCN_REQUIRE(a->first >= 0 && (long long)a->first + a->B <= a->num_frustums,
                "frustums [first, first + B) outside the segment table");
    if (a->B == 0) return FCN_OK;
    FCN_REQUIRE(a->dataset == FCN_DET_KITTI || a->NS >= 1, "SUN-RGBD scores need NS >= 1");
    FCN_REQUIRE(a->cls_probs && a->center && a->heading && a->size && a->rot_angle && a->seg_of_frustum &&
                    a->counter && (a->records || a->capacity == 0) && (a->dataset == FCN_DET_KITTI || a->size_probs),
                "NULL pointer");
    det_candidates_kernel<<<a->B, DET_THREADS, 0, (cudaStream_t)stream>>>(*a);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

extern "C" long long fcn_det_workspace_bytes(int capacity, int num_segments) {
    if (capacity < 0 || num_segments < 0 || num_segments >= (1 << 20)) {
        invalid(__func__, "bad sizes (capacity >= 0, 0 <= num_segments < 2^20)");
        return -1;
    }
    DetWs w;
    return workspace_size(__func__, [&](Carve &c) { return det_layout(std::max(capacity, 1), num_segments, c, w); });
}

static int det_check_finalize(const fcn_det_finalize_args *a, const char *fn) {
    if (a == nullptr) return invalid(fn, "NULL args");
    if (a->num_segments < 0 || a->num_segments >= (1 << 20) || a->capacity < 0 || a->num_frustums < 0 ||
        a->top_k < 1)
        return invalid(fn, "bad sizes (0 <= num_segments < 2^20, capacity >= 0, top_k >= 1)");
    if (a->method != FCN_DET_NMS && a->method != FCN_DET_TOP) return invalid(fn, "method must be 0 (nms) or 1 (top)");
    if (a->dataset != FCN_DET_KITTI && a->dataset != FCN_DET_SUNRGBD)
        return invalid(fn, "dataset must be 0 (KITTI) or 1 (SUN-RGBD)");
    if (!a->counter || !a->info || !a->seg_offsets || !a->keep_count || !a->workspace ||
        (a->capacity > 0 && (!a->records || !a->rows || !a->box2d)))
        return invalid(fn, "NULL pointer");
    return FCN_OK;
}

extern "C" int fcn_det_prepare(const fcn_det_finalize_args *a, fcn_stream_t stream) {
    int st = det_check_finalize(a, __func__);
    if (st != FCN_OK) return st;
    const int C = std::max(a->capacity, 1), S = a->num_segments, nms = a->method == FCN_DET_NMS;
    cudaStream_t s = (cudaStream_t)stream;
    DetWs w;
    st = carve_workspace(__func__, "det", a->workspace, a->workspace_bytes,
                         [&](Carve &c) { return det_layout(C, S, c, w); });
    if (st != FCN_OK) return st;
    FCN_CUDA(cudaMemsetAsync(w.seg_cnt, 0, (size_t)(S + 1) * 4, s));
    const int g = det_grid(C, DET_FIN_THREADS);
    det_keys_kernel<<<g, DET_FIN_THREADS, 0, s>>>(a->capacity, a->counter, a->records, w.keys_a, w.vals_a, w.seg_cnt);
    FCN_LAUNCH_CHECK();
    if (a->capacity > 0) {
        FCN_CUDA(cub::DeviceRadixSort::SortPairs(w.temp, w.temp_bytes, w.keys_a, w.keys_b, w.vals_a, w.vals_b,
                                                 a->capacity, 0, 64, s));
        det_gather_sorted_kernel<<<g, DET_FIN_THREADS, 0, s>>>(a->capacity, a->counter, nms, a->records, w.vals_b,
                                                               w.sorted, w.keys_a, w.vals_a);
        FCN_LAUNCH_CHECK();
        if (nms) {
            // rank sort: stable ascending (segment, score); read backwards per segment = descending score, ties
            // larger list index first (the reverse of a stable ascending sort, oracle/nms.py)
            FCN_CUDA(cub::DeviceRadixSort::SortPairs(w.temp, w.temp_bytes, w.keys_a, w.keys_b, w.vals_a, w.vals_b,
                                                     a->capacity, 0, 64, s));
        }
    }
    FCN_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, w.temp_bytes, w.seg_cnt, a->seg_offsets, S + 1, s));
    det_seg_sizes_kernel<<<det_grid(S + 1, DET_FIN_THREADS), DET_FIN_THREADS, 0, s>>>(S, nms, w.seg_cnt, w.mask_w,
                                                                                      w.tiles);
    FCN_LAUNCH_CHECK();
    FCN_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, w.temp_bytes, w.mask_w, w.mask_off, S + 1, s));
    FCN_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, w.temp_bytes, w.tiles, w.tile_off, S + 1, s));
    det_info_kernel<<<1, 1, 0, s>>>(S, a->counter, w.mask_off, w.tile_off, a->info);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

extern "C" int fcn_det_select(const fcn_det_finalize_args *a, fcn_stream_t stream) {
    int st = det_check_finalize(a, __func__);
    if (st != FCN_OK) return st;
    if (a->n_counted < 0 || a->n_counted > a->capacity) {
        snprintf(g_err, sizeof(g_err),
                 "%s: record capacity exceeded: %d rows were produced, the capacity is %d (needs capacity >= %d)",
                 __func__, a->n_counted, a->capacity, a->n_counted);
        return FCN_ERR_INVALID;
    }
    const int C = std::max(a->capacity, 1), S = a->num_segments, n = a->n_counted, nms = a->method == FCN_DET_NMS;
    cudaStream_t s = (cudaStream_t)stream;
    DetWs w;
    st = carve_workspace(__func__, "det", a->workspace, a->workspace_bytes,
                         [&](Carve &c) { return det_layout(C, S, c, w); });
    if (st != FCN_OK) return st;
    FCN_REQUIRE(!nms || a->mask_words >= 0, "bad mask_words");
    FCN_REQUIRE(!nms || a->mask_words == 0 || a->mask, "NULL mask");
    if (n > 0 && nms) {
        det_rank_kernel<<<det_grid(n, DET_FIN_THREADS), DET_FIN_THREADS, 0, s>>>(n, w.sorted, a->seg_offsets,
                                                                                 w.vals_b, w.rank_idx, w.corners,
                                                                                 w.cube);
        FCN_LAUNCH_CHECK();
        if (a->mask_words > 0) {
            det_pairs_kernel<<<sm_count() * 8, DET_FIN_THREADS, 0, s>>>(S, a->thresh, a->seg_offsets, w.mask_off,
                                                                        w.tile_off, w.corners, w.cube, a->mask);
            FCN_LAUNCH_CHECK();
        }
        FCN_CUDA(cudaMemsetAsync(w.removed, 0, ((size_t)n / 32 + (size_t)S + 2) * 4, s));
    }
    if (S > 0) {
        det_scan_kernel<<<det_grid((long long)S * 32, DET_FIN_THREADS), DET_FIN_THREADS, 0, s>>>(
            S, nms, a->top_k, a->seg_offsets, w.mask_off, a->mask, w.removed, w.keep, a->keep_count);
        FCN_LAUNCH_CHECK();
    }
    if (n > 0) {
        det_rows_kernel<<<det_grid(n, DET_FIN_THREADS), DET_FIN_THREADS, 0, s>>>(
            n, nms, a->dataset, w.sorted, a->seg_offsets, w.rank_idx, w.keep, a->keep_count, a->box2d, a->rows);
        FCN_LAUNCH_CHECK();
    }
    return FCN_OK;
}
