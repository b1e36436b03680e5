// Sliding-frustum grouping kernels.
//
//  * qdp_kernel        — drop-in for query_depth_point_gpu
//                        (/root/reference/ops/query_depth_point/query_depth_point_cuda_kernel.cu:16-65):
//                        one WARP per (frustum, section) instead of one thread; 32 points are tested
//                        per step with ballot/popc compaction, so idx stores are contiguous and the
//                        z reads are coalesced.  Bit-exact: same fp32 `fabsf(z2 - z1) < dis_z`
//                        predicate, same first-K-in-index-order selection, same back-fill.
//  * group_rows_kernel — fused form used by the PointNet tile kernels: no int64 idx tensor is
//                        materialised; each section emits float4 {x-cx, y-cy, z-cz, t} row records
//                        (gather + centre subtraction of models/det_base.py:75-80 folded in).
#include "common.cuh"

namespace fcn {

thread_local char g_err[512] = "";

int sm_count() {   // per device: a process may drive several GPUs (ADVICE r1)
    static int cache[64] = {0};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    int n = cache[dev];
    if (n == 0) {
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 148;
        cache[dev] = n;
    }
    return n;
}

// The predicate of cu:48-53.  __fsub_rn / fabsf keep it a plain IEEE fp32 subtract (no contraction).
__device__ __forceinline__ bool depth_hit(float zc, float zp, float dis_z) {
    return fabsf(__fsub_rn(zc, zp)) < dis_z;
}

constexpr int QDP_WARPS = 8;

template <bool CHANNEL_FIRST>
__global__ void __launch_bounds__(QDP_WARPS * 32)
qdp_kernel(int n, int m, float dis_z, int nsample, const float *__restrict__ xyz1,
           const float *__restrict__ xyz2, long long *__restrict__ idx, int *__restrict__ pts_cnt) {
    const int b = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int sec = blockIdx.x * QDP_WARPS + warp;
    if (sec >= m) return;
    const float *z1;
    int zstride;
    float zc;
    if (CHANNEL_FIRST) {
        z1 = xyz1 + (size_t)b * 3 * n + 2 * (size_t)n;
        zstride = 1;
        zc = __ldg(xyz2 + (size_t)b * 3 * m + 2 * (size_t)m + sec);
    } else {
        z1 = xyz1 + (size_t)b * n * 3 + 2;
        zstride = 3;
        zc = __ldg(xyz2 + ((size_t)b * m + sec) * 3 + 2);
    }
    long long *out = idx + ((size_t)b * m + sec) * nsample;
    int cnt = 0, first = 0;
    for (int base = 0; base < n && cnt < nsample; base += 32) {
        const int k = base + lane;
        bool hit = false;
        if (k < n) hit = depth_hit(zc, __ldg(z1 + (size_t)k * zstride), dis_z);
        const unsigned mask = __ballot_sync(0xffffffffu, hit);
        if (mask) {
            if (cnt == 0) first = base + __ffs(mask) - 1;
            const int pos = cnt + __popc(mask & ((1u << lane) - 1));
            if (hit && pos < nsample) out[pos] = k;
            cnt += __popc(mask);
        }
    }
    cnt = min(cnt, nsample);
    // back-fill (cu:55-59): slots >= cnt repeat the first hit; empty sections stay all-zero
    for (int l = cnt + lane; l < nsample; l += 32) out[l] = first;
    if (lane == 0) pts_cnt[(size_t)b * m + sec] = cnt;
}

// ---------------------------------------------------------------------------------------------
// Fused grouping, two launches:
//   group_count_kernel : grid (section chunks, S, B), one warp per section, 4 independent 32-point
//                        ballots in flight per step; writes cnt (B,T) and the first min(hits,K) point
//                        indices (int32 scratch, same order as the reference idx tensor).
//   group_emit_kernel  : grid (B, S): block scan of cnt -> row offsets, tile table, zero-filled
//                        feature block + one-hot channels, then one warp per section gathers
//                        {x-cx, y-cy, z-cz, t} row records (no second scan of the cloud).
struct GroupParams {
    fcn_group_args a;
};

constexpr int GC_WARPS = 32;           // sections per CTA in group_count_kernel
constexpr int GE_THREADS = 512;

__global__ void __launch_bounds__(GC_WARPS * 32)
group_count_kernel(const __grid_constant__ GroupParams P) {
    const fcn_group_args &a = P.a;
    const int b = blockIdx.y;
    pdl_wait();
    pdl_launch_dependents();
    // the tile counters of this forward are reset here (group_emit_kernel runs after this grid)
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x < FCN_MAX_SCALES) a.ntiles[threadIdx.x] = 0;
    // blockIdx.x enumerates (scale, 32-section chunk) pairs
    int s = 0, chunk = blockIdx.x;
    for (; s < a.num_scales; ++s) {
        const int nc = ceil_div(a.T[s], GC_WARPS);
        if (chunk < nc) break;
        chunk -= nc;
    }
    if (s >= a.num_scales) return;
    const int N = a.N, T = a.T[s], K = a.K[s];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int t0 = chunk * GC_WARPS;
    // this CTA owns the feature rows of its 32 sections: zero them and write the one-hot channels
    // (det_base.py:145-157) here, where 600+ CTAs share the 11.5 MB instead of one CTA per (b, scale)
    if (a.feat[s] != nullptr) {
        const int ld = a.ld_feat[s], c3 = a.c3[s], V = a.num_vec;
        const int nt = min(GC_WARPS, T - t0);
        const int fp = a.feat_pitch[s] > 0 ? a.feat_pitch[s] : T;
        float4 *f4 = (float4 *)(a.feat[s] + ((size_t)b * fp + t0) * ld);
        const int n4 = nt * ld / 4;
        const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int i = threadIdx.x; i < n4; i += blockDim.x) f4[i] = z4;
        if (a.one_hot != nullptr && V > 0) {
            __syncthreads();
            float *fb = a.feat[s] + ((size_t)b * fp + t0) * ld;
            for (int i = threadIdx.x; i < nt * V; i += blockDim.x) {
                const int t = i / V, v = i - t * V;
                fb[(size_t)t * ld + c3 + v] = __ldg(a.one_hot + (size_t)b * V + v);
            }
        }
    }
    const int t = t0 + warp;
    if (t >= T) return;
    // one warp per section; the z row is read straight from global memory (coalesced, L1-resident for the
    // 32 warps of the CTA), four independent 32-point ballots in flight per step
    const float *pz = a.pc + (size_t)b * 3 * N + 2 * (size_t)N;
    const float dis_z = a.dis_z[s];
    const float zc = __ldg(a.centers[s] + (size_t)b * 3 * T + 2 * (size_t)T + t);
    int *out = a.idx_scratch[s] + ((size_t)b * T + t) * K;
    const unsigned lt = (1u << lane) - 1u;
    int cnt = 0;
    for (int base = 0; base < N && cnt < K; base += 128) {
        float zv[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = base + j * 32 + lane;
            zv[j] = k < N ? __ldg(pz + k) : 0.f;
        }
        bool hit[4];
        unsigned m[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            hit[j] = (base + j * 32 + lane < N) && depth_hit(zc, zv[j], dis_z);
            m[j] = __ballot_sync(0xffffffffu, hit[j]);
        }
        if ((m[0] | m[1] | m[2] | m[3]) == 0u) continue;   // most 128-point steps miss a narrow section
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int pos = cnt + __popc(m[j] & lt);
            if (hit[j] && pos < K) out[pos] = base + j * 32 + lane;
            cnt += __popc(m[j]);
        }
    }
    if (lane == 0) a.cnt[s][(size_t)b * T + t] = min(cnt, K);
}

__global__ void __launch_bounds__(GE_THREADS)
group_emit_kernel(const __grid_constant__ GroupParams P) {
    extern __shared__ int sm_i[];
    const fcn_group_args &a = P.a;
    const int b = blockIdx.x, s = blockIdx.y;
    const int N = a.N, T = a.T[s], K = a.K[s];
    int *scnt = sm_i, *sstart = sm_i + T;
    float *scen = (float *)(sm_i + 2 * T);     // 3T: section centres (x | y | z)
    __shared__ int s_warp_tot[GE_THREADS / 32];
    __shared__ int s_carry, s_total, s_tile_base;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    pdl_wait();
    pdl_launch_dependents();
    const int *gcnt = a.cnt[s] + (size_t)b * T;
    for (int i = threadIdx.x; i < T; i += blockDim.x) scnt[i] = gcnt[i];
    {
        const float *cen_g = a.centers[s] + (size_t)b * 3 * T;
        for (int i = threadIdx.x; i < 3 * T; i += blockDim.x) scen[i] = __ldg(cen_g + i);
    }
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    const bool uniq = a.unique_rows != 0;
    for (int base = 0; base < T; base += blockDim.x) {
        const int t = base + threadIdx.x;
        int v = 0;
        if (t < T) v = uniq ? scnt[t] : K;
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int u = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += u;
        }
        if (lane == 31) s_warp_tot[warp] = incl;
        __syncthreads();
        int woff = 0;
        for (int w = 0; w < warp; ++w) woff += s_warp_tot[w];
        const int carry = s_carry;
        if (t < T) sstart[t] = carry + woff + incl - v;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) s_carry = carry + woff + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const int total = s_carry;
        s_total = total;
        const int nt = ceil_div(total, a.tile_rows);
        s_tile_base = nt > 0 ? atomicAdd(a.ntiles + s, nt) : 0;
    }
    __syncthreads();
    const int total = s_total;
    {
        int4 *tiles = (int4 *)a.tiles[s];
        const int nt = ceil_div(total, a.tile_rows);
        for (int i = threadIdx.x; i < nt; i += blockDim.x) {
            const int row0 = i * a.tile_rows;
            if (s_tile_base + i < a.tile_cap[s])
                tiles[s_tile_base + i] = make_int4(b, row0, min(a.tile_rows, total - row0), 0);
        }
    }
    // row records, one thread per row (independent gathers -> latency overlapped)
    const float *px = a.pc + (size_t)b * 3 * N, *py = px + N, *pz = py + N;
    float4 *rows = (float4 *)a.rows[s] + (size_t)b * a.row_cap[s];
    const int *gidx = a.idx_scratch[s] + (size_t)b * T * K;
    const int nrows_total = uniq ? total : T * K;
    for (int i = threadIdx.x; i < nrows_total; i += blockDim.x) {
        int t, l;
        if (uniq) {   // upper_bound over the exclusive offsets: last t with sstart[t] <= i and cnt > 0
            int lo = 0, hi = T - 1;
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (sstart[mid] <= i) lo = mid; else hi = mid - 1;
            }
            t = lo;
            l = i - sstart[t];
        } else {
            t = i / K;
            l = i - t * K;
        }
        const int c = scnt[t];
        const int k = c > 0 ? gidx[(size_t)t * K + (l < c ? l : 0)] : 0;   // back-fill: first hit (cu:55-59)
        const int tag = c > 0 ? t : (t | 0x80000000);
        rows[i] = make_float4(__fsub_rn(__ldg(px + k), scen[t]), __fsub_rn(__ldg(py + k), scen[T + t]),
                              __fsub_rn(__ldg(pz + k), scen[2 * T + t]), __int_as_float(tag));
    }
}

// ---------------------------------------------------------------------------------------------
// Fused grouping, single launch (used whenever the hit bitmasks of one (frustum, scale) fit in shared
// memory): instead of letting every section scan all N points (N*T predicate evaluations per scale —
// group_count_kernel is issue-bound), every POINT marks the sections it falls into in a T x N bit matrix:
//   phase 1  thread per point: when the section centres are sorted (the data providers emit them in
//            ascending depth) a binary search finds the first centre >= z and the exact fp32 predicate is
//            walked left/right from there (the hit set is contiguous for sorted centres because the rounded
//            difference is monotone); unsorted centres fall back to testing all T sections.  Hits are
//            atomicOr'ed into the section's row of the bit matrix.
//   phase 2  warp per section: popcount prefix over the row's words gives every hit its rank in ascending
//            point order — exactly the order of the reference's serial scan (cu:42-63); cnt = min(hits, K).
//   then     block scan of cnt -> row offsets, tile table, zero-filled feature rows + one-hot, row records.
// Same outputs (rows, tiles, cnt, feat) as group_count_kernel + group_emit_kernel, bit-exact.
constexpr int GB_THREADS = 1024;

__global__ void __launch_bounds__(GB_THREADS)
group_bitmask_kernel(const __grid_constant__ GroupParams P) {
    extern __shared__ unsigned sm_u[];
    const fcn_group_args &a = P.a;
    const int b = blockIdx.x, s = blockIdx.y;
    const int N = a.N, T = a.T[s], K = a.K[s];
    const int W = (N + 31) >> 5;                       // words per section row
    unsigned *bm = sm_u;                               // T * W
    float *zc = (float *)(bm + (size_t)T * W);         // T
    int *scnt = (int *)(zc + T), *sstart = scnt + T;   // T, T
    __shared__ int s_warp_tot[GB_THREADS / 32];
    __shared__ int s_carry, s_total, s_tile_base;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nwarp = blockDim.x >> 5;
    pdl_wait();
    pdl_launch_dependents();
    const float dis_z = a.dis_z[s];
    const float *pz = a.pc + (size_t)b * 3 * N + 2 * (size_t)N;
    const float *cen = a.centers[s] + (size_t)b * 3 * T;
    for (int i = tid; i < T * W; i += blockDim.x) bm[i] = 0u;
    for (int i = tid; i < T; i += blockDim.x) zc[i] = __ldg(cen + 2 * T + i);
    if (tid == 0) s_carry = 0;
    __syncthreads();
    int sorted = 1;
    for (int i = tid; i + 1 < T; i += blockDim.x) sorted &= (zc[i + 1] >= zc[i]) ? 1 : 0;   // NaN -> unsorted
    sorted = __syncthreads_and(sorted);

    // ---- phase 1: points -> bit matrix
    for (int k = tid; k < N; k += blockDim.x) {
        const float z = __ldg(pz + k);
        const unsigned bit = 1u << (k & 31);
        unsigned *col = bm + (k >> 5);
        if (sorted) {
            int lo = 0, hi = T;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (zc[mid] < z) lo = mid + 1; else hi = mid;
            }
            for (int t = lo - 1; t >= 0 && depth_hit(zc[t], z, dis_z); --t) atomicOr(col + (size_t)t * W, bit);
            for (int t = lo; t < T && depth_hit(zc[t], z, dis_z); ++t) atomicOr(col + (size_t)t * W, bit);
        } else {
            for (int t = 0; t < T; ++t)
                if (depth_hit(zc[t], z, dis_z)) atomicOr(col + (size_t)t * W, bit);
        }
    }
    __syncthreads();
    // ---- phase 2a: hits per section
    for (int t = warp; t < T; t += nwarp) {
        int c = 0;
        for (int w = lane; w < W; w += 32) c += __popc(bm[(size_t)t * W + w]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0) scnt[t] = min(c, K);
    }
    __syncthreads();
    // ---- exclusive scan of rows-per-section
    const bool uniq = a.unique_rows != 0;
    for (int base = 0; base < T; base += blockDim.x) {
        const int t = base + tid;
        int v = 0;
        if (t < T) v = uniq ? scnt[t] : K;
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int u = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += u;
        }
        if (lane == 31) s_warp_tot[warp] = incl;
        __syncthreads();
        int woff = 0;
        for (int w = 0; w < warp; ++w) woff += s_warp_tot[w];
        const int carry = s_carry;
        if (t < T) sstart[t] = carry + woff + incl - v;
        __syncthreads();
        if (tid == blockDim.x - 1) s_carry = carry + woff + incl;
        __syncthreads();
    }
    if (tid == 0) {
        const int total = s_carry;
        s_total = total;
        const int nt = ceil_div(total, a.tile_rows);
        s_tile_base = nt > 0 ? atomicAdd(a.ntiles + s, nt) : 0;
    }
    __syncthreads();
    const int total = s_total;
    {
        int4 *tiles = (int4 *)a.tiles[s];
        const int nt = ceil_div(total, a.tile_rows);
        for (int i = tid; i < nt; i += blockDim.x) {
            const int row0 = i * a.tile_rows;
            if (s_tile_base + i < a.tile_cap[s])
                tiles[s_tile_base + i] = make_int4(b, row0, min(a.tile_rows, total - row0), 0);
        }
        int *gcnt = a.cnt[s] + (size_t)b * T;
        for (int i = tid; i < T; i += blockDim.x) gcnt[i] = scnt[i];
    }
    if (a.feat[s] != nullptr) {   // zero-filled feature rows + one-hot channels (det_base.py:145-157)
        const int ld = a.ld_feat[s], c3 = a.c3[s], V = a.num_vec;
        const int fp = a.feat_pitch[s] > 0 ? a.feat_pitch[s] : T;
        float *fb = a.feat[s] + (size_t)b * fp * ld;
        float4 *f4 = (float4 *)fb;
        const int n4 = T * ld / 4;
        const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int i = tid; i < n4; i += blockDim.x) f4[i] = z4;
        if (a.one_hot != nullptr && V > 0) {
            __syncthreads();
            for (int i = tid; i < T * V; i += blockDim.x) {
                const int t = i / V, v = i - t * V;
                fb[(size_t)t * ld + c3 + v] = __ldg(a.one_hot + (size_t)b * V + v);
            }
        }
    }
    // ---- phase 2b: rank every hit (popcount prefix inside the section's row = ascending point order) and park
    //      its point index in shared memory; then one thread per row gathers and writes the record
    //      (independent loads, coalesced 16-byte stores)
    int *rowk = sstart + T;                            // row_cap ints
    for (int t = warp; t < T; t += nwarp) {
        const int c = scnt[t];
        if (c == 0) continue;
        int *dst = rowk + sstart[t];
        int done = 0;
        for (int wb = 0; wb < W && done < K; wb += 32) {
            const int w = wb + lane;
            unsigned word = w < W ? bm[(size_t)t * W + w] : 0u;
            const int n = __popc(word);
            int incl = n;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                int u = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += u;
            }
            int pos = done + incl - n;
            while (word && pos < K) {
                dst[pos++] = w * 32 + __ffs(word) - 1;
                word &= word - 1;
            }
            done += __shfl_sync(0xffffffffu, incl, 31);
        }
    }
    __syncthreads();
    const float *px = a.pc + (size_t)b * 3 * N, *py = px + N;
    float4 *rows = (float4 *)a.rows[s] + (size_t)b * a.row_cap[s];
    const int nrows_total = uniq ? total : T * K;
    for (int i = tid; i < nrows_total; i += blockDim.x) {
        int t, l;
        if (uniq) {   // last t with sstart[t] <= i (empty sections share the offset of their successor)
            int lo = 0, hi = T - 1;
            while (lo < hi) {
                const int mid = (lo + hi + 1) >> 1;
                if (sstart[mid] <= i) lo = mid; else hi = mid - 1;
            }
            t = lo;
            l = i - sstart[t];
        } else {
            t = i / K;
            l = i - t * K;
        }
        const int c = scnt[t];
        // reference back-fill (cu:55-59): slots >= cnt repeat the first hit; masked sections gather point 0
        const int k = c > 0 ? rowk[sstart[t] + (l < c ? l : 0)] : 0;
        const int tag = c > 0 ? t : (t | 0x80000000);
        rows[i] = make_float4(__fsub_rn(__ldg(px + k), __ldg(cen + t)), __fsub_rn(__ldg(py + k), __ldg(cen + T + t)),
                              __fsub_rn(__ldg(pz + k), zc[t]), __int_as_float(tag));
    }
}

// ntiles reset for the single-launch path (a tiny grid in front of group_bitmask_kernel)
__global__ void group_reset_kernel(int32_t *ntiles) {
    pdl_wait();
    pdl_launch_dependents();
    if (threadIdx.x < FCN_MAX_SCALES) ntiles[threadIdx.x] = 0;
}

}  // namespace fcn

using namespace fcn;

extern "C" int fcn_version(void) { return 100; }
extern "C" const char *fcn_last_error(void) { return fcn::g_err; }

static int qdp_launch(bool channel_first, int b, int n, int m, float dis_z, int nsample,
                      const float *xyz1, const float *xyz2, int64_t *idx, int32_t *pts_cnt,
                      fcn_stream_t stream) {
    FCN_REQUIRE(b >= 0 && n >= 0 && m >= 0, "negative size");
    FCN_REQUIRE(nsample > 0, "nsample must be positive");
    FCN_REQUIRE(b <= 65535, "batch exceeds gridDim.y");
    if (b == 0 || m == 0) return FCN_OK;
    FCN_REQUIRE(xyz1 || n == 0, "xyz1 is NULL");
    FCN_REQUIRE(xyz2 && idx && pts_cnt, "NULL pointer");
    dim3 grid(ceil_div(m, QDP_WARPS), b), block(QDP_WARPS * 32);
    if (channel_first)
        qdp_kernel<true><<<grid, block, 0, (cudaStream_t)stream>>>(
            n, m, dis_z, nsample, xyz1, xyz2, (long long *)idx, pts_cnt);
    else
        qdp_kernel<false><<<grid, block, 0, (cudaStream_t)stream>>>(
            n, m, dis_z, nsample, xyz1, xyz2, (long long *)idx, pts_cnt);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

extern "C" int fcn_query_depth_point_bn3(int b, int n, int m, float dis_z, int nsample,
                                         const float *xyz1, const float *xyz2, int64_t *idx,
                                         int32_t *pts_cnt, fcn_stream_t stream) {
    return qdp_launch(false, b, n, m, dis_z, nsample, xyz1, xyz2, idx, pts_cnt, stream);
}
extern "C" int fcn_query_depth_point_b3n(int b, int n, int m, float dis_z, int nsample,
                                         const float *xyz1, const float *xyz2, int64_t *idx,
                                         int32_t *pts_cnt, fcn_stream_t stream) {
    return qdp_launch(true, b, n, m, dis_z, nsample, xyz1, xyz2, idx, pts_cnt, stream);
}

extern "C" int fcn_group_rows(const fcn_group_args *args, fcn_stream_t stream) {
    FCN_REQUIRE(args != nullptr, "args is NULL");
    const fcn_group_args &a = *args;
    FCN_REQUIRE(a.num_scales >= 1 && a.num_scales <= FCN_MAX_SCALES, "num_scales out of range");
    FCN_REQUIRE(a.B >= 0 && a.N >= 1, "bad B/N");
    FCN_REQUIRE(a.tile_rows >= 1, "tile_rows must be positive");
    FCN_REQUIRE(a.pc && a.ntiles, "NULL pointer");
    if (a.B == 0) return FCN_OK;
    int maxT = 0;
    for (int s = 0; s < a.num_scales; ++s) {
        FCN_REQUIRE(a.T[s] >= 1 && a.K[s] >= 1, "bad T/K");
        FCN_REQUIRE(a.centers[s] && a.rows[s] && a.cnt[s] && a.tiles[s], "NULL per-scale pointer");
        // checked on both paths: only the section-scan pair uses it, but which pair runs depends on the shape
        FCN_REQUIRE(a.idx_scratch[s] != nullptr, "NULL idx_scratch");
        FCN_REQUIRE(a.row_cap[s] >= a.T[s] * a.K[s], "row_cap too small");
        FCN_REQUIRE(a.feat[s] == nullptr || a.ld_feat[s] % 4 == 0, "ld_feat must be a multiple of 4");
        FCN_REQUIRE(a.feat[s] == nullptr || a.ld_feat[s] >= a.c3[s] + a.num_vec, "ld_feat too small");
        maxT = a.T[s] > maxT ? a.T[s] : maxT;
    }
    GroupParams P;
    P.a = a;
    // single-launch bit-matrix path when T x N bits (+ 3T words) of the largest scale fit in shared memory
    size_t smem_b = 0;
    for (int s = 0; s < a.num_scales; ++s) {
        const size_t need = sizeof(unsigned) * ((size_t)a.T[s] * ((a.N + 31) / 32) + 3 * (size_t)a.T[s] +
                                                (size_t)a.T[s] * a.K[s]);
        smem_b = need > smem_b ? need : smem_b;
    }
    const bool force_scan = a.force_scan != 0;   // A-B testing of the two grouping paths (host decides)
    FCN_REQUIRE(a.B <= 65535 && a.num_scales <= 65535, "grid too large");
    if (smem_b <= 200 * 1024 && !force_scan) {
        if (smem_b > 48 * 1024)
            FCN_CUDA(cudaFuncSetAttribute(group_bitmask_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_b));
        FCN_CUDA(launch_pdl(group_reset_kernel, dim3(1), dim3(32), (size_t)0, (cudaStream_t)stream, a.ntiles));
        FCN_CUDA(launch_pdl(group_bitmask_kernel, dim3(a.B, a.num_scales), dim3(GB_THREADS), smem_b,
                            (cudaStream_t)stream, P));
        return FCN_OK;
    }
    const size_t smem_e = sizeof(int) * 5 * (size_t)maxT;
    FCN_REQUIRE(smem_e <= 200 * 1024, "T too large for the shared-memory staging");
    if (smem_e > 48 * 1024)
        FCN_CUDA(cudaFuncSetAttribute(group_emit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_e));
    int nchunks = 0;
    for (int s = 0; s < a.num_scales; ++s) nchunks += ceil_div(a.T[s], GC_WARPS);
    dim3 gc(nchunks, a.B);
    FCN_CUDA(launch_pdl(group_count_kernel, gc, dim3(GC_WARPS * 32), (size_t)0, (cudaStream_t)stream, P));
    dim3 ge(a.B, a.num_scales);
    FCN_CUDA(launch_pdl(group_emit_kernel, ge, dim3(GE_THREADS), smem_e, (cudaStream_t)stream, P));
    return FCN_OK;
}
