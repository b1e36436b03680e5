// PointNet tile kernel, TF32 tensor-core variant ("precision = 1"): wgmma (TF32 in, fp32 accumulators in
// registers), weight tiles staged by the TMA engine (1-D bulk copies of pre-swizzled images, mbarrier ring).
//
// Per 128-row tile (rows = unique grouped points {dx,dy,dz,section} from group_rows_kernel), two compute
// warpgroups each own 64 rows and run the whole chain on them without waiting for each other:
//   layer 1 (3->C1, fp32 FMA, folded BN, ReLU) -> A operand in shared memory (K-major, 128B swizzle, TF32)
//   layer 2 D2[64 x C2] = A1 * W2^T (wgmma) -> +bias, ReLU, TF32 -> A2 (same rows of the same buffer)
//   layer 3 D3[64 x 128-channel chunk] = A2 * W3^T -> +bias, ReLU, max over the rows of each section:
//           a segmented suffix max over the 16 rows of a warp (shuffles), then one integer atomicMax per
//           (section part, channel) into the position-major feature map
// A loader warp streams (or keeps resident) the pre-swizzled W2/W3 stage images; both warpgroups read
// every stage, and a stage is released when both have retired the wgmma group that read it.
//
// "precision = 2" runs the same kernel on clusters of two CTAs (CL = 2, streamed-weight scales only): the two
// CTAs take the two tiles of a tile pair in lock step, and every weight stage is fetched from L2 ONCE per
// cluster - each CTA's loader copies one half of it with a multicast bulk copy into both CTAs.  A stage slot is
// refilled only when the consumer warps of BOTH CTAs have released it (remote mbarrier arrivals).
#include "common.cuh"
#include "wgmma.cuh"

namespace fcn {
using namespace gmma;

constexpr int TC_ROWS = 128;
constexpr int TC_COMPUTE_WARPS = 8;                         // two warpgroups of 64 tile rows each
constexpr int TC_THREADS = (TC_COMPUTE_WARPS + 1) * 32;     // + the weight loader warp
constexpr int TC_STAGE_BYTES = 16384;

template <int C1, int C2, int C3>
struct TcCfg {
    static constexpr int KB1 = C1 / 32, KB2 = C2 / 32;
    static constexpr int N2 = C2 < 128 ? C2 : 128;
    static constexpr int NCH2 = C2 / N2;
    static constexpr int N3 = 128;
    static constexpr int NCH3 = C3 / N3;
    static constexpr int A_BYTES = TC_ROWS * (C1 > C2 ? C1 : C2) * 4;
    static constexpr int JOBS2 = NCH2 * KB1, JOBS3 = NCH3 * KB2, JOBS = JOBS2 + JOBS3;
    // streamed rings: at C1 = 256, 4 stages measured faster on an H100 than 3 or 5 (5 is the most that fits)
    static constexpr int NSTAGE = (C1 >= 256) ? 4 : (C1 >= 128 ? 6 : JOBS);
    static constexpr bool RESIDENT = JOBS <= NSTAGE;
    // Small-channel scales are latency-bound per tile (tiny MMAs, long SIMT phases): run TWO CTAs per SM
    // so that one CTA's epilogue overlaps the other's loads/MMAs.
    static constexpr int CTAS_PER_SM = (C1 <= 64) ? 2 : 1;
    static constexpr int OFF_W = A_BYTES;
    // resident weights are packed tightly (layer-2 stages are only N2 x 128 B), streamed stages use 16 KB slots
    static constexpr int W_BYTES = RESIDENT ? (JOBS2 * N2 * 128 + JOBS3 * TC_STAGE_BYTES) : NSTAGE * TC_STAGE_BYTES;
    __host__ __device__ static constexpr int stage_off(int st) {
        return !RESIDENT ? st * TC_STAGE_BYTES
                         : (st < JOBS2 ? st * N2 * 128 : JOBS2 * N2 * 128 + (st - JOBS2) * TC_STAGE_BYTES);
    }
    static constexpr int OFF_RECS = OFF_W + W_BYTES;
    static constexpr int OFF_W1 = OFF_RECS + 2 * TC_ROWS * 16;       // recs are double-buffered by tile parity
    static constexpr int OFF_B2 = OFF_W1 + C1 * 16;
    static constexpr int OFF_B3 = OFF_B2 + C2 * 4;
    static constexpr int OFF_SECT = OFF_B3 + C3 * 4;                 // int sect[2][128]
    static constexpr int OFF_BAR = OFF_SECT + 2 * TC_ROWS * 4;
    static constexpr int NBAR = 2 * NSTAGE;
    static constexpr int BYTES = OFF_BAR + NBAR * 8 + 1024;          // + alignment slack
    static_assert(C1 % 32 == 0 && C2 % 32 == 0 && C3 % 128 == 0, "channel counts");
    static_assert(C2 <= 256, "layer-2 accumulators: at most two 128-column chunks");
    static_assert(BYTES <= 232448, "exceeds the 227 KB shared-memory limit per CTA");
    static_assert(CTAS_PER_SM == 1 || 2 * (BYTES + 1024) <= 233472, "two CTAs must fit in 228 KB per SM");
};

template <int C1, int C2, int C3, int CL>
__global__ void __launch_bounds__(TC_THREADS, (TcCfg<C1, C2, C3>::CTAS_PER_SM))
pointnet_tc_kernel(const __grid_constant__ fcn_pointnet_args p) {
    using Cfg = TcCfg<C1, C2, C3>;
    static_assert(CL == 1 || (CL == 2 && !Cfg::RESIDENT), "2-CTA clusters share streamed weight stages");
    extern __shared__ uint8_t smem_dyn[];
    uint8_t *smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
    uint8_t *sA = smem;
    uint8_t *sW = smem + Cfg::OFF_W;
    float4 *recs_all = (float4 *)(smem + Cfg::OFF_RECS);
    float4 *w1s = (float4 *)(smem + Cfg::OFF_W1);
    float *b2s = (float *)(smem + Cfg::OFF_B2);
    float *b3s = (float *)(smem + Cfg::OFF_B3);
    int *sect_all = (int *)(smem + Cfg::OFF_SECT);
    uint64_t *bars = (uint64_t *)(smem + Cfg::OFF_BAR);
    uint64_t *w_full = bars, *w_empty = bars + Cfg::NSTAGE;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    pdl_wait();                 // tile table / rows / feature map come from the grouping kernels
    pdl_launch_dependents();
    const int ntiles = min(*p.ntiles, p.max_tiles);
    // Work unit = CL consecutive tiles, one per CTA of the cluster (unit u, rank r: tile u * CL + r; a rank without
    // a tile in the last unit runs it with zero rows so that both CTAs stream the same weight stages).
    // Unit stride of the persistent loop: the cluster count, or (FCN_BALANCE_ROUNDS) only as many clusters as the
    // round count needs - e.g. 2.4 rounds become 3 rounds on 80 % of the clusters, the rest exit at once and
    // leave their SMs to the kernels of the other in-flight forwards.  The decision is uniform per cluster.
    const int rank = CL == 2 ? (int)cluster_ctarank() : 0;
    const int cid = (int)blockIdx.x / CL, units = (ntiles + CL - 1) / CL;
    const int tstride = balanced_stride(units, (int)gridDim.x / CL);
    if (cid >= units || cid >= tstride) return;  // whole cluster exits: nothing was started
    const int my_tiles = (units - cid + tstride - 1) / tstride;
    auto tile_of = [&](int it) {                 // tile descriptor of round `it` (nrows = 0: no tile)
        const int tix = (cid + it * tstride) * CL + rank;
        return tix < ntiles ? ((const int4 *)p.tiles)[tix] : make_int4(0, 0, 0, 0);
    };

    // ---- one-time setup
    for (int i = tid; i < C1; i += TC_THREADS)
        w1s[i] = make_float4(__ldg(p.w1t + i), __ldg(p.w1t + C1 + i), __ldg(p.w1t + 2 * C1 + i), __ldg(p.b1 + i));
    for (int i = tid; i < C2; i += TC_THREADS) b2s[i] = __ldg(p.b2 + i);
    for (int i = tid; i < C3; i += TC_THREADS) b3s[i] = __ldg(p.b3 + i);
    if (tid == 0) {
        for (int i = 0; i < Cfg::NSTAGE; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], TC_COMPUTE_WARPS * CL); }
        fence_barrier_init();
    }
    __syncthreads();
    if (CL == 2) cluster_sync();                 // the peer's barriers are initialised before anyone signals them

    if (warp == TC_COMPUTE_WARPS) {
        // ================= weight loader (one lane) =================
        if (lane == 0) {
            const int ntile_loads = Cfg::RESIDENT ? 1 : my_tiles;
            uint32_t job = 0;
            for (int it = 0; it < ntile_loads; ++it) {
                for (int j = 0; j < Cfg::JOBS; ++j, ++job) {
                    const uint32_t st = job % Cfg::NSTAGE, ph = (job / Cfg::NSTAGE) & 1;
                    mbar_wait(&w_empty[st], ph ^ 1);   // CL = 2: released by the consumers of both CTAs
                    const bool l2 = j < Cfg::JOBS2;
                    const uint32_t bytes = l2 ? Cfg::N2 * 128 : TC_STAGE_BYTES;
                    const uint8_t *src = l2 ? (const uint8_t *)p.w2_tc + (size_t)j * (Cfg::N2 * 128)
                                            : (const uint8_t *)p.w3_tc + (size_t)(j - Cfg::JOBS2) * TC_STAGE_BYTES;
                    mbar_arrive_expect_tx(&w_full[st], bytes);   // both halves land on this CTA's barrier
                    if (CL == 2) {
                        const uint32_t half = bytes / 2, off = (uint32_t)rank * half;
                        bulk_g2s_multicast(sW + Cfg::stage_off(st) + off, src + off, half, &w_full[st], 0x3);
                    } else {
                        bulk_g2s(sW + Cfg::stage_off(st), src, bytes, &w_full[st]);
                    }
                }
            }
        }
    } else {

        // ================= compute warpgroups =================
        const int wg = warp >> 2, wq = warp & 3, t = tid & 127;
        const int l1_row = 64 * wg + (t & 63);                 // layer-1 role: row, K blocks kb = t/64, t/64 + 2, ...
        const uint32_t l1_off = (uint32_t)((l1_row >> 3) * 1024 + (l1_row & 7) * 128);
        const int rx = l1_row & 7;
        const uint64_t adesc0 = make_desc_sw128(smem_u32(sA) + wg * (64 * 128));
        const uint64_t bdesc0 = make_desc_sw128(smem_u32(sW));
        const int ra = 64 * wg + 16 * wq + (lane >> 2);        // fragment rows of this thread: ra and ra + 8
        uint32_t job = 0;
        int4 td_next = tile_of(0);
        float4 rec_next = make_float4(0.f, 0.f, 0.f, 0.f);
        if (tid < TC_ROWS && tid < td_next.z)
            rec_next = ((const float4 *)p.rows + (size_t)td_next.x * p.row_cap + td_next.y)[tid];

        // one weight stage per call: wait, 4 wgmma (k = 8 each), commit; the stage of the previous call is released
        // once its group has retired (streamed weights only)
        int prev = -1;
        auto release_prev = [&]() {
            if (!Cfg::RESIDENT && prev >= 0 && lane == 0) {
                if (CL == 2) {
                    mbar_arrive_cluster(&w_empty[prev], 0);
                    mbar_arrive_cluster(&w_empty[prev], 1);
                } else {
                    mbar_arrive(&w_empty[prev]);
                }
            }
            prev = -1;
        };

        for (int it = 0; it < my_tiles; ++it) {
            const int4 td = td_next;           // tile descriptor + the staged record were prefetched
            const int b = td.x, nrows = td.z;  // during the previous tile (two dependent global loads)
            // staging buffers alternate with the tile parity: a warp that runs ahead into tile it+1
            // must not overwrite what slower warps still read for tile it (they meet at this barrier)
            float4 *recs = recs_all + (it & 1) * TC_ROWS;
            int *sect_s = sect_all + (it & 1) * TC_ROWS;
            if (tid < TC_ROWS) {
                recs[tid] = rec_next;
                sect_s[tid] = tid < nrows ? (__float_as_int(rec_next.w) & 0x7fffffff) : -1;
            }
            if (it + 1 < my_tiles) {
                td_next = tile_of(it + 1);
                rec_next = make_float4(0.f, 0.f, 0.f, 0.f);
                if (tid < TC_ROWS && tid < td_next.z)
                    rec_next = ((const float4 *)p.rows + (size_t)td_next.x * p.row_cap + td_next.y)[tid];
            }
            asm volatile("bar.sync 1, %0;\n" ::"n"(TC_COMPUTE_WARPS * 32));
            const float4 rec = recs[l1_row];
            // ---- layer 1 (fp32 FMA) -> A1
            for (int kb = t >> 6; kb < Cfg::KB1; kb += 2) {
                uint8_t *dst = sA + kb * (TC_ROWS * 128) + l1_off;
    #pragma unroll
                for (int c4 = 0; c4 < 8; ++c4) {
                    float o[4];
    #pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float4 w = w1s[kb * 32 + c4 * 4 + j];
                        o[j] = to_tf32(fmaxf(fmaf(rec.z, w.z, fmaf(rec.y, w.y, fmaf(rec.x, w.x, w.w))), 0.f));
                    }
                    *(float4 *)(dst + ((c4 ^ rx) << 4)) = make_float4(o[0], o[1], o[2], o[3]);
                }
            }
            fence_proxy_async();
            asm volatile("bar.sync %0, 128;\n" ::"r"(2 + wg));
            if (Cfg::RESIDENT) job = 0;

            // ---- layer 2: D2 = A1 * W2^T, all NCH2 chunks in registers (A2 overwrites A1)
            float acc2[Cfg::NCH2][Cfg::N2 / 2];
    #pragma unroll
            for (int nc = 0; nc < Cfg::NCH2; ++nc) {
    #pragma unroll
                for (int i = 0; i < Cfg::N2 / 2; ++i) acc2[nc][i] = 0.f;
                for (int kb = 0; kb < Cfg::KB1; ++kb, ++job) {
                    const uint32_t st = job % Cfg::NSTAGE, ph = Cfg::RESIDENT ? 0 : (job / Cfg::NSTAGE) & 1;
                    mbar_wait(&w_full[st], ph);
                    wgmma_fence();
                    fence_acc(acc2[nc]);
    #pragma unroll
                    for (int k = 0; k < 4; ++k)
                        wgmma_tf32<Cfg::N2>(acc2[nc], adesc0 + (uint64_t)(kb * ((TC_ROWS * 128) >> 4) + 2 * k),
                                            bdesc0 + (uint64_t)((Cfg::stage_off(st) >> 4) + 2 * k), (kb | k) != 0);
                    wgmma_commit();
                    fence_acc(acc2[nc]);
                    if (!Cfg::RESIDENT) {
                        wgmma_wait<1>();
                        release_prev();
                        prev = (int)st;
                    }
                }
            }
            wgmma_wait<0>();
    #pragma unroll
            for (int nc = 0; nc < Cfg::NCH2; ++nc) fence_acc(acc2[nc]);
            release_prev();
            // ---- epilogue 2: +bias, ReLU, TF32 -> A2 (this warpgroup's rows; all its layer-2 MMAs are done)
    #pragma unroll
            for (int nc = 0; nc < Cfg::NCH2; ++nc)
    #pragma unroll
                for (int i = 0; i < Cfg::N2 / 2; i += 2) {
                    const int r = 64 * wg + frag_row(i, wq, lane), c = nc * Cfg::N2 + frag_col(i, lane);
                    const float2 bb = *(const float2 *)(b2s + c);
                    const float2 o = make_float2(to_tf32(fmaxf(acc2[nc][i] + bb.x, 0.f)),
                                                 to_tf32(fmaxf(acc2[nc][i + 1] + bb.y, 0.f)));
                    *(float2 *)(sA + (c >> 5) * (TC_ROWS * 128) + sw128_offset(r, c & 31)) = o;
                }
            fence_proxy_async();
            asm volatile("bar.sync %0, 128;\n" ::"r"(2 + wg));

            // ---- layer 3 + section max.  Rows ra (fragment half 0) and ra + 8 (half 1) of this thread; the suffix
            //      max over the rows of a section runs over the 8 lanes l/4 = 0..7 of each half, then half 0 takes in
            //      half 1's head when the section crosses row 8 of the warp.  +bias, ReLU, TF32 rounding commute with
            //      the max (monotone), values >= 0 so the integer atomicMax on the float bits is exact.
            const int g = lane >> 2;
            const int sa = sect_s[ra], sb = sect_s[ra + 8], s8 = sect_s[ra - g + 8];
            unsigned oka = 0, okb = 0;                 // bit d: row + (1 << d) is in the same section and 8-row half
    #pragma unroll
            for (int d = 0; d < 3; ++d) {
                const int o = 1 << d;
                if (g + o < 8 && sa >= 0 && sect_s[ra + o] == sa) oka |= 1u << d;
                if (g + o < 8 && sb >= 0 && sect_s[ra + 8 + o] == sb) okb |= 1u << d;
            }
            const bool merge_a = sa >= 0 && sa == s8;
            const bool head_a = sa >= 0 && (g == 0 || sect_s[ra - 1] != sa);
            const bool head_b = sb >= 0 && sect_s[ra + 7] != sb;
            int *feat = (int *)(p.out + (size_t)b * p.feat_pitch * p.ld_feat);
            for (int nc = 0; nc < Cfg::NCH3; ++nc) {
                float acc3[Cfg::N3 / 2];
    #pragma unroll
                for (int i = 0; i < Cfg::N3 / 2; ++i) acc3[i] = 0.f;
                for (int kb = 0; kb < Cfg::KB2; ++kb, ++job) {
                    const uint32_t st = job % Cfg::NSTAGE, ph = Cfg::RESIDENT ? 0 : (job / Cfg::NSTAGE) & 1;
                    mbar_wait(&w_full[st], ph);
                    wgmma_fence();
                    fence_acc(acc3);
    #pragma unroll
                    for (int k = 0; k < 4; ++k)
                        wgmma_tf32<Cfg::N3>(acc3, adesc0 + (uint64_t)(kb * ((TC_ROWS * 128) >> 4) + 2 * k),
                                            bdesc0 + (uint64_t)((Cfg::stage_off(st) >> 4) + 2 * k), (kb | k) != 0);
                    wgmma_commit();
                    fence_acc(acc3);
                    if (!Cfg::RESIDENT) {
                        wgmma_wait<1>();
                        release_prev();
                        prev = (int)st;
                    }
                }
                wgmma_wait<0>();
                fence_acc(acc3);
                release_prev();
    #pragma unroll
                for (int j = 0; j < Cfg::N3 / 8; ++j) {
                    float v[4] = {acc3[4 * j], acc3[4 * j + 1], acc3[4 * j + 2], acc3[4 * j + 3]};
    #pragma unroll
                    for (int d = 0; d < 3; ++d) {
    #pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const float x = __shfl_down_sync(0xffffffffu, v[e], 4 << d);
                            if (((e < 2 ? oka : okb) >> d) & 1u) v[e] = fmaxf(v[e], x);
                        }
                    }
    #pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float x = __shfl_sync(0xffffffffu, v[2 + e], lane & 3);   // row 8 of this warp
                        if (merge_a) v[e] = fmaxf(v[e], x);
                    }
                    const int c = nc * Cfg::N3 + 8 * j + 2 * (lane & 3);
                    const float2 bb = *(const float2 *)(b3s + c);
    #pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const bool head = e < 2 ? head_a : head_b;
                        const float o = to_tf32(v[e] + ((e & 1) ? bb.y : bb.x));
                        if (head && o > 0.f)
                            atomicMax(feat + (size_t)(e < 2 ? sa : sb) * p.ld_feat + c + (e & 1), __float_as_int(o));
                    }
                }
            }
        }
    }
    if (CL == 2) {                               // the peer may still signal this CTA's barriers
        __syncwarp();
        cluster_sync();
    }
}

template <int C1, int C2, int C3, int CL>
static int launch_tc(const fcn_pointnet_args &a, cudaStream_t stream) {
    using Cfg = TcCfg<C1, C2, C3>;
    auto kern = pointnet_tc_kernel<C1, C2, C3, CL>;
    FCN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::BYTES));
    int clusters = sm_count() * Cfg::CTAS_PER_SM / CL;
    if (clusters > (a.max_tiles + CL - 1) / CL) clusters = (a.max_tiles + CL - 1) / CL;
    if (clusters < 1) return FCN_OK;
    static const int prio = env_priority("FCN_PRIO_PN");
    FCN_CUDA(launch_pdl_cluster(prio, CL, kern, dim3(clusters * CL), dim3(TC_THREADS), (size_t)Cfg::BYTES, stream, a));
    return FCN_OK;
}

int pointnet_tiles_tc(const fcn_pointnet_args &a, cudaStream_t stream) {
    FCN_REQUIRE(a.tile_rows == TC_ROWS, "the TF32 tensor-core variant needs tile_rows == 128");
    FCN_REQUIRE(!a.unpooled, "the tensor-core variant only produces the pooled feature map");
    FCN_REQUIRE(a.w2_tc && a.w3_tc, "NULL tensor-core weight image");
    if (a.precision == 2) {
        if (a.C1 == 128 && a.C2 == 128 && a.C3 == 256) return launch_tc<128, 128, 256, 2>(a, stream);
        if (a.C1 == 256 && a.C2 == 256 && a.C3 == 512) return launch_tc<256, 256, 512, 2>(a, stream);
        return invalid("fcn_pointnet_tiles",
                       "unsupported (C1,C2,C3) for 2-CTA clusters; built: (128,128,256) (256,256,512)");
    }
    if (a.C1 == 64 && a.C2 == 64 && a.C3 == 128) return launch_tc<64, 64, 128, 1>(a, stream);
    if (a.C1 == 128 && a.C2 == 128 && a.C3 == 256) return launch_tc<128, 128, 256, 1>(a, stream);
    if (a.C1 == 256 && a.C2 == 256 && a.C3 == 512) return launch_tc<256, 256, 512, 1>(a, stream);
    return invalid("fcn_pointnet_tiles",
                   "unsupported (C1,C2,C3); built: (64,64,128) (128,128,256) (256,256,512)");
}

}  // namespace fcn
