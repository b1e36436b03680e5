// PointNet tile kernel, TF32 tensor-core variant ("precision = 1"): wgmma (TF32 in, fp32 accumulators in
// registers), weight tiles staged by the TMA engine (1-D bulk copies of pre-swizzled images, mbarrier ring).
//
// Per 128-row tile (rows = unique grouped points {dx,dy,dz,section} from group_rows_kernel), two compute
// warpgroups each own 64 rows and run the whole chain on them in registers, without waiting for each other:
//   layer 1 (3->C1, fp32 FMA, folded BN, ReLU, TF32) -> straight into the A fragments of layer 2 (8 columns per
//           k-step, double-buffered by K block so that it runs under the previous block's MMAs)
//   layer 2 D2[64 x C2] = A1 * W2^T (wgmma, A from registers) -> +bias, ReLU, TF32 in place, then an intra-quad
//           permutation turns the accumulator fragments into the A fragments of layer 3 (resident for the tile)
//   layer 3 D3[64 x N3-channel chunk] = A2 * W3^T (A from registers) -> +bias, ReLU, max over the rows of each
//           section part in a warp's 16 rows, then one integer atomicMax per (section part, channel) into the
//           position-major feature map.  A warp takes one masked reduce-scatter pass over its lanes per section
//           that starts in its rows (7 shuffles per 32 channels and section, one coalesced atomic per lane).
// Only the weights go through shared memory.  A loader warp streams (or keeps resident) the pre-swizzled W2/W3
// stage images; both warpgroups read every stage, and a stage is released when both have retired the wgmma group
// that read it.  The loader is a whole warpgroup that gives its registers to the two consumer warpgroups
// (setmaxnreg): at C2 = 256 the layer-3 A fragments alone take 128 registers per thread.
//
// "precision = 2" runs the same kernel on clusters of two CTAs (CL = 2, streamed-weight scales only): the two
// CTAs take the two tiles of a tile pair in lock step, and every weight stage is fetched from L2 ONCE per
// cluster - each CTA's loader copies one half of it with a multicast bulk copy into both CTAs.  A stage slot is
// refilled only when the consumer warps of BOTH CTAs have released it (remote mbarrier arrivals).
#include "common.cuh"
#include "wgmma.cuh"

// Streamed weight ring at C1 = 256, in 16 KB stages (A-B builds: -DFCN_PN_RING_C256=N).
#ifndef FCN_PN_RING_C256
#define FCN_PN_RING_C256 4
#endif

namespace fcn {
using namespace gmma;

constexpr int TC_ROWS = 128;
constexpr int TC_COMPUTE_WARPS = 8;                         // two warpgroups of 64 tile rows each
constexpr int TC_STAGE_BYTES = 16384;
constexpr int TC_SMEM_MAX = 232448;                         // 227 KB of dynamic shared memory per CTA

template <int C1, int C2, int C3, int CL>
struct TcCfg {
    static constexpr int KB1 = C1 / 32, KB2 = C2 / 32;
    static constexpr int N2 = C2 < 128 ? C2 : 128;
    static constexpr int NCH2 = C2 / N2;
    // W2 stage images in load order: K block major, its NCH2 column chunks side by side (job kb * NCH2 + nc)
    static constexpr int JOBS2 = NCH2 * KB1, JOBS3 = (C3 / 128) * KB2, JOBS = JOBS2 + JOBS3;
    // Small-channel scales are latency-bound per tile (tiny MMAs, long SIMT phases): run TWO CTAs per SM
    // so that one CTA's epilogue overlaps the other's loads/MMAs.
    static constexpr int CTAS_PER_SM = (C1 <= 64) ? 2 : 1;
    // + the loader warpgroup (one lane loads), which gives its registers to the consumers: the layer-3 A fragments
    // alone take C2 / 2 registers per thread.  One CTA per SM: 168 at launch -> 232 / 40 (2 x 232 + 40 per lane of
    // an SM sub-partition); two CTAs per SM: 80 at launch -> 104 / 24 (8 x 104 + 4 x 24 = 12 x 80 per CTA).
    static constexpr int THREADS = (TC_COMPUTE_WARPS + 4) * 32;
    static constexpr int REGS_CONSUMER = CTAS_PER_SM == 1 ? 232 : 104, REGS_PRODUCER = CTAS_PER_SM == 1 ? 40 : 24;
    static constexpr int OTHER_BYTES = 2 * TC_ROWS * 16 + C1 * 16 + C2 * 4 + C3 * 4 + 2 * TC_ROWS * 4;
    // weight-resident when every stage fits (packed tightly: layer-2 stages are only N2 x 128 B); 2-CTA clusters
    // exist to share streamed stages
    static constexpr int W_RES_BYTES = JOBS2 * N2 * 128 + JOBS3 * TC_STAGE_BYTES;
    static constexpr bool RESIDENT =
        CL == 1 && W_RES_BYTES + OTHER_BYTES + 2 * JOBS * 8 + 1024 <= TC_SMEM_MAX / CTAS_PER_SM - (CTAS_PER_SM - 1) * 1024;
    // streamed rings: 6 stages at C1 = 128 (2-CTA clusters only), 4 at C1 = 256 (with the activations in registers,
    // car pointnet_s4 measured 0.101-0.103 ms per launch with 4, 8 and 12 stages alike on an H100 SXM at 400 W)
    static constexpr int NSTAGE = RESIDENT ? JOBS : (C1 >= 256 ? FCN_PN_RING_C256 : 6);
    // layer-3 chunk: 64 channels at two CTAs per SM (the register budget is 96 per thread there), else 128; a
    // 64-channel chunk reads one half of a 128-row W3 stage image (resident weights only)
    static constexpr int N3 = CTAS_PER_SM == 2 ? 64 : 128;
    static constexpr int SUB3 = 128 / N3, NCH3 = C3 / N3;
    static constexpr int W_BYTES = RESIDENT ? W_RES_BYTES : NSTAGE * TC_STAGE_BYTES;
    __host__ __device__ static constexpr int stage_off(int st) {
        return !RESIDENT ? st * TC_STAGE_BYTES
                         : (st < JOBS2 ? st * N2 * 128 : JOBS2 * N2 * 128 + (st - JOBS2) * TC_STAGE_BYTES);
    }
    static constexpr int OFF_W = 0;
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
    static_assert(N3 == 128 || RESIDENT, "64-channel layer-3 chunks read resident W3 stages");
    static_assert(BYTES <= TC_SMEM_MAX, "exceeds the 227 KB shared-memory limit per CTA");
    static_assert(CTAS_PER_SM == 1 || 2 * (BYTES + 1024) <= 233472, "two CTAs must fit in 228 KB per SM");
};

// One layer-1 output (fp32 FMA chain, folded BN, ReLU) as a TF32 operand.
__device__ __forceinline__ uint32_t layer1_tf32(const float4 &r, const float4 &w) {
    return __float_as_uint(to_tf32(fmaxf(fmaf(r.z, w.z, fmaf(r.y, w.y, fmaf(r.x, w.x, w.w))), 0.f)));
}

// Max over the 16 rows of a warp that belong to ONE section, for the 32 columns of accumulator blocks
// j0 .. j0 + 3 (acc[4j + e]: rows ra (e < 2) and ra + 8 (e >= 2), columns 8j + 2q + (e & 1)).  in_a / in_b: row ra /
// ra + 8 is in the section; any other row (another section, or past nrows, whose staged record is zero-filled)
// becomes -inf by a select before any fmaxf.  The 8 values of a thread are reduce-scattered over the 8 lanes g = 0..7 that share
// q (butterfly over lane bits 16, 8, 4: each level keeps one half and receives the partner's max of the other half,
// 4 + 2 + 1 shuffles), so lane g ends up with the section max of value g, i.e. column 8 (j0 + g / 2) + 2q + g % 2;
// then +bias, TF32 and one integer atomicMax if positive.  dst / bias point at column 0 of
// the chunk.  32 columns at a time keep the temporaries at 8 registers next to the A fragments and accumulators.
template <int H>            // one butterfly level over lane bit 4H: 2H values in, H out
__device__ __forceinline__ void max_scatter_level(float (&v)[8], int lane) {
    const bool hi = (lane & (4 * H)) != 0;
#pragma unroll
    for (int i = 0; i < H; ++i) {
        const float send = hi ? v[i] : v[i + H], keep = hi ? v[i + H] : v[i];
        v[i] = fmaxf(keep, __shfl_xor_sync(0xffffffffu, send, 4 * H));
    }
}

template <int R>
__device__ __forceinline__ void section_max_32(const float (&acc)[R], int j0, bool in_a, bool in_b, int *dst,
                                               const float *bias, int lane) {
    float v[8];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            const float x = in_a ? acc[4 * (j0 + j) + c] : -INFINITY;
            const float y = in_b ? acc[4 * (j0 + j) + 2 + c] : -INFINITY;
            v[2 * j + c] = fmaxf(x, y);
        }
    max_scatter_level<4>(v, lane);
    max_scatter_level<2>(v, lane);
    max_scatter_level<1>(v, lane);
    const int g = lane >> 2, c = 8 * (j0 + (g >> 1)) + 2 * (lane & 3) + (g & 1);
    const float o = to_tf32(v[0] + bias[c]);
    if (o > 0.f) atomicMax(dst + c, __float_as_int(o));
}

template <int C1, int C2, int C3, int CL>
__global__ void __launch_bounds__((TcCfg<C1, C2, C3, CL>::THREADS), (TcCfg<C1, C2, C3, CL>::CTAS_PER_SM))
pointnet_tc_kernel(const __grid_constant__ fcn_pointnet_args p) {
    using Cfg = TcCfg<C1, C2, C3, CL>;
    static_assert(CL == 1 || (CL == 2 && !Cfg::RESIDENT), "2-CTA clusters share streamed weight stages");
    extern __shared__ uint8_t smem_dyn[];
    uint8_t *smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
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
    for (int i = tid; i < C1; i += Cfg::THREADS)
        w1s[i] = make_float4(__ldg(p.w1t + i), __ldg(p.w1t + C1 + i), __ldg(p.w1t + 2 * C1 + i), __ldg(p.b1 + i));
    for (int i = tid; i < C2; i += Cfg::THREADS) b2s[i] = __ldg(p.b2 + i);
    for (int i = tid; i < C3; i += Cfg::THREADS) b3s[i] = __ldg(p.b3 + i);
    if (tid == 0) {
        for (int i = 0; i < Cfg::NSTAGE; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], TC_COMPUTE_WARPS * CL); }
        fence_barrier_init();
    }
    __syncthreads();
    if (CL == 2) cluster_sync();                 // the peer's barriers are initialised before anyone signals them

    if (warp >= TC_COMPUTE_WARPS) {
        // ================= weight loader (one lane of the loader warpgroup) =================
        setmaxnreg_dec<Cfg::REGS_PRODUCER>();
        if (warp == TC_COMPUTE_WARPS && lane == 0) {
            const int ntile_loads = Cfg::RESIDENT ? 1 : my_tiles;
            uint32_t job = 0;
            for (int it = 0; it < ntile_loads; ++it) {
                for (int j = 0; j < Cfg::JOBS; ++j, ++job) {
                    const uint32_t st = job % Cfg::NSTAGE, ph = (job / Cfg::NSTAGE) & 1;
                    mbar_wait(&w_empty[st], ph ^ 1);   // CL = 2: released by the consumers of both CTAs
                    const bool l2 = j < Cfg::JOBS2;
                    const uint32_t bytes = l2 ? Cfg::N2 * 128 : TC_STAGE_BYTES;
                    // the W2 image is chunk major (chunk nc, K block kb at nc * KB1 + kb)
                    const int j2 = (j % Cfg::NCH2) * Cfg::KB1 + j / Cfg::NCH2;
                    const uint8_t *src = l2 ? (const uint8_t *)p.w2_tc + (size_t)j2 * (Cfg::N2 * 128)
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
        setmaxnreg_inc<Cfg::REGS_CONSUMER>();
        const int wg = warp >> 2, wq = warp & 3;
        const int g = lane >> 2, q = lane & 3;
        const int ra = 64 * wg + 16 * wq + g;                  // fragment rows of this thread: ra and ra + 8
        const uint64_t bdesc0 = make_desc_sw128(smem_u32(sW));
        // Layer-2 accumulators -> layer-3 A fragments.  In each 8-column block, lane q of a quad holds columns
        // (2q, 2q + 1) and needs (q, q + 4).  Two shuffles move the quad's 8 values: in the first, lane q sends
        // its column 2q + psel and receives from lane src1; in the second it sends the other one and receives from
        // src1 ^ 2.  Lanes with psel = 0 receive column q first, lanes with psel = 1 column q + 4.
        const int psel = (q ^ (q >> 1)) & 1;
        const int src1 = (lane & ~3) | (q >> 1) | (psel << 1), src2 = src1 ^ 2;
        // Each warpgroup stages its own 64 rows (threads 0..63 of the warpgroup, row srow) into the record / section
        // buffers of the tile parity.  Tile it + 1's record is loaded before tile it's barrier and stored at the end of
        // tile it, so that the two dependent global loads have the whole tile to land; at C2 = 256 the layer-3 A
        // fragments leave no registers to hold it through layer 3, so it is stored once layer 2 has run.
        constexpr bool STAGE_AFTER_L2 = C2 > 128;
        const bool stager = (tid & 64) == 0;
        const int srow = 64 * wg + (tid & 63);
        auto load_rec = [&](const int4 &t) {
            return stager && srow < t.z ? ((const float4 *)p.rows + (size_t)t.x * p.row_cap + t.y)[srow]
                                        : make_float4(0.f, 0.f, 0.f, 0.f);
        };
        auto stage_rec = [&](int parity, const float4 &r, int nrows) {
            if (stager) {
                recs_all[parity * TC_ROWS + srow] = r;
                sect_all[parity * TC_ROWS + srow] = srow < nrows ? (__float_as_int(r.w) & 0x7fffffff) : -1;
            }
        };
        uint32_t job = 0;
        int4 td_next = tile_of(0);
        stage_rec(0, load_rec(td_next), td_next.z);

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
            const int b = td_next.x;           // tile descriptor + the staged record were prefetched
                                               // during the previous tile (two dependent global loads)
            // The staging buffers alternate with the tile parity.  Tile it + 1's buffer is written after this
            // barrier, which every warp of the warpgroup reaches only once it has read tile it - 1's; a warpgroup
            // reads only its own rows, so the two warpgroups never wait for each other here and may drift apart by
            // up to the weight ring's depth.
            const float4 *recs = recs_all + (it & 1) * TC_ROWS;
            const int *sect_s = sect_all + (it & 1) * TC_ROWS;
            float4 rec_next;
            if (it + 1 < my_tiles) {
                td_next = tile_of(it + 1);
                rec_next = load_rec(td_next);
            }
            asm volatile("bar.sync %0, 128;\n" ::"r"(2 + wg));
            const float4 reca = recs[ra], recb = recs[ra + 8];
            if (Cfg::RESIDENT) job = 0;

            // ---- layers 1 + 2: per K block, layer 1 computes the A fragments of its 4 k-steps (columns
            //      32 kb + 8 k + q and + 4 of rows ra, ra + 8) while the previous block's MMAs run; D2 = A1 * W2^T
            //      for all NCH2 chunks in registers.  The fragments alternate between two buffers: a buffer is
            //      rewritten two K blocks later, after wait_group 1 has retired every group that read it.
            float acc2[Cfg::NCH2][Cfg::N2 / 2];
    #pragma unroll
            for (int nc = 0; nc < Cfg::NCH2; ++nc)
    #pragma unroll
                for (int i = 0; i < Cfg::N2 / 2; ++i) acc2[nc][i] = 0.f;
            uint32_t a1[2][4][4];
    #pragma unroll
            for (int kb = 0; kb < Cfg::KB1; ++kb) {
                uint32_t (&a)[4][4] = a1[kb & 1];
    #pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float4 w0 = w1s[kb * 32 + 8 * k + q], w4 = w1s[kb * 32 + 8 * k + q + 4];
                    a[k][0] = layer1_tf32(reca, w0);
                    a[k][1] = layer1_tf32(recb, w0);
                    a[k][2] = layer1_tf32(reca, w4);
                    a[k][3] = layer1_tf32(recb, w4);
                    fence_frag(a[k]);
                }
    #pragma unroll
                for (int nc = 0; nc < Cfg::NCH2; ++nc, ++job) {
                    const uint32_t st = job % Cfg::NSTAGE, ph = Cfg::RESIDENT ? 0 : (job / Cfg::NSTAGE) & 1;
                    mbar_wait(&w_full[st], ph);
                    wgmma_fence();
                    fence_acc(acc2[nc]);
    #pragma unroll
                    for (int k = 0; k < 4; ++k)
                        wgmma_tf32_rs<Cfg::N2>(acc2[nc], a[k], bdesc0 + (uint64_t)((Cfg::stage_off(st) >> 4) + 2 * k),
                                               (kb | k) != 0);
                    wgmma_commit();
                    fence_acc(acc2[nc]);
                    wgmma_wait<1>();
                    release_prev();
                    prev = (int)st;
                }
            }
            wgmma_wait<0>();
    #pragma unroll
            for (int nc = 0; nc < Cfg::NCH2; ++nc) fence_acc(acc2[nc]);
            release_prev();
            if (STAGE_AFTER_L2 && it + 1 < my_tiles) stage_rec((it + 1) & 1, rec_next, td_next.z);
            // ---- epilogue 2: +bias, ReLU, TF32 in place, then the quad permutation into the A fragments of the
            //      KB2 * 4 k-steps of layer 3 (k-step s = columns 8 s .. 8 s + 7)
            uint32_t a2[Cfg::KB2 * 4][4];
    #pragma unroll
            for (int nc = 0; nc < Cfg::NCH2; ++nc)
    #pragma unroll
                for (int j = 0; j < Cfg::N2 / 8; ++j) {
                    const float2 bb = *(const float2 *)(b2s + nc * Cfg::N2 + 8 * j + 2 * q);
    #pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const float v0 = to_tf32(fmaxf(acc2[nc][4 * j + 2 * h] + bb.x, 0.f));
                        const float v1 = to_tf32(fmaxf(acc2[nc][4 * j + 2 * h + 1] + bb.y, 0.f));
                        const float x1 = __shfl_sync(0xffffffffu, psel ? v1 : v0, src1);
                        const float x2 = __shfl_sync(0xffffffffu, psel ? v0 : v1, src2);
                        uint32_t (&a)[4] = a2[nc * (Cfg::N2 / 8) + j];
                        a[h] = __float_as_uint(psel ? x2 : x1);
                        a[2 + h] = __float_as_uint(psel ? x1 : x2);
                    }
                }
    #pragma unroll
            for (int s = 0; s < Cfg::KB2 * 4; ++s) fence_frag(a2[s]);

            // ---- layer 3 + section max.  Warp-uniform shape of the warp's 16 rows: sections are contiguous runs and
            //      the rows past nrows (sect -1) a suffix, so the rows that start a section give the warp's sections;
            //      each takes its own section_max_32 passes (1 or 2 sections in almost every warp at C1 >= 128, up to
            //      16 at the small scales).  +bias, ReLU, TF32 rounding commute with the max (monotone), values >= 0
            //      so the integer atomicMax on the float bits is exact.
            int *feat = (int *)(p.out + (size_t)b * p.feat_pitch * p.ld_feat);
            for (int nc = 0; nc < Cfg::NCH3; ++nc) {
                float acc3[Cfg::N3 / 2];
    #pragma unroll
                for (int i = 0; i < Cfg::N3 / 2; ++i) acc3[i] = 0.f;
    #pragma unroll
                for (int kb = 0; kb < Cfg::KB2; ++kb, ++job) {
                    // resident: W3 stage (128-channel chunk nc / SUB3, K block kb), column half nc % SUB3
                    const uint32_t st = Cfg::RESIDENT ? Cfg::JOBS2 + (nc / Cfg::SUB3) * Cfg::KB2 + kb : job % Cfg::NSTAGE;
                    const uint32_t ph = Cfg::RESIDENT ? 0 : (job / Cfg::NSTAGE) & 1;
                    const uint32_t boff = Cfg::stage_off(st) + (nc % Cfg::SUB3) * (Cfg::N3 * 128);
                    mbar_wait(&w_full[st], ph);
                    wgmma_fence();
                    fence_acc(acc3);
    #pragma unroll
                    for (int k = 0; k < 4; ++k)
                        wgmma_tf32_rs<Cfg::N3>(acc3, a2[4 * kb + k], bdesc0 + (uint64_t)((boff >> 4) + 2 * k),
                                               (kb | k) != 0);
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
                // the warp's section shape (re-read per chunk from shared memory rather than held in registers
                // through the MMAs): bit i of `starts` marks row i of the warp's 16 as the first of a section in
                // them (row 0 whenever it is below nrows); the rows past nrows (sect -1) start nothing
                const int sa = sect_s[ra], sb = sect_s[ra + 8];
                const int r0 = ra - g, rl = r0 + (lane & 15);
                const int sl = sect_s[rl];
                unsigned starts =
                    __ballot_sync(0xffffffffu, lane < 16 && sl >= 0 && (lane == 0 || sl != sect_s[rl - 1]));
                const int c0 = nc * Cfg::N3;
                while (starts) {                       // one reduce-scatter pass per section, 0..16 of them
                    const int s = __shfl_sync(0xffffffffu, sl, __ffs(starts) - 1);
                    starts &= starts - 1;
    #pragma unroll
                    for (int h = 0; h < Cfg::N3 / 32; ++h)
                        section_max_32(acc3, 4 * h, sa == s, sb == s, feat + (size_t)s * p.ld_feat + c0, b3s + c0,
                                       lane);
                }
            }
            if (!STAGE_AFTER_L2 && it + 1 < my_tiles) stage_rec((it + 1) & 1, rec_next, td_next.z);
        }
    }
    if (CL == 2) {                               // the peer may still signal this CTA's barriers
        __syncwarp();
        cluster_sync();
    }
}

template <int C1, int C2, int C3, int CL>
static int launch_tc(const fcn_pointnet_args &a, cudaStream_t stream) {
    using Cfg = TcCfg<C1, C2, C3, CL>;
    auto kern = pointnet_tc_kernel<C1, C2, C3, CL>;
    FCN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::BYTES));
    int clusters = sm_count() * Cfg::CTAS_PER_SM / CL;
    if (clusters > (a.max_tiles + CL - 1) / CL) clusters = (a.max_tiles + CL - 1) / CL;
    if (clusters < 1) return FCN_OK;
    static const int prio = env_priority("FCN_PRIO_PN");
    FCN_CUDA(launch_pdl_cluster(prio, CL, kern, dim3(clusters * CL), dim3(Cfg::THREADS), (size_t)Cfg::BYTES, stream, a));
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
