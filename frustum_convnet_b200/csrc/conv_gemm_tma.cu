// Implicit-GEMM conv on wgmma with a fully TMA-fed pipeline ("precision = 3|4").
//
// Same math as conv_gemm_tc.cu; differs in how the A operand reaches shared memory: instead of the LDGSTS
// gather of that kernel, every [128 positions x 32 channels] atom is ONE cp.async.bulk.tensor (TMA) box of a
// 3-D tensor map (channel, position, frustum) with hardware 128-byte swizzle.  An M tile is 128
// consecutive rows of the flattened (frustum, padded position) sequence (the maps are encoded with B = 1,
// T = frustums x pitch), so
//   * kernel taps are a coordinate offset (t*stride + tap, may be -1): the zero pad row(s) that follow every
//     frustum, and the TMA unit's zero fill before the first and after the last row, ARE the conv zero padding
//     (nn.Conv1d(..., padding=1)); a tap never reaches the neighbouring frustum's rows;
//   * stride-2 convs use the map's elementStrides (box 256 -> 128 loaded rows);
//   * channels past ld and the K padding blocks are zero-filled by the TMA unit.
// One elected thread issues A boxes + the weight bulk copy of a 64-wide K stage onto ONE mbarrier; two
// consumer warpgroups (64 rows each) issue 8 wgmma per stage and store their accumulators.  No proxy fence,
// no producer warps.
#include <cuda.h>

#include "common.cuh"
#include "conv_epilogue.cuh"
#include "wgmma.cuh"

namespace fcn {
using namespace gmma;

constexpr int GM_ROWS = 128;
constexpr int GM_MMA_WARPS = 8;                  // warps 0-7: two consumer warpgroups; warp 8: TMA producer
constexpr int GM_THREADS = (GM_MMA_WARPS + 1) * 32;

template <int NT>
struct GmCfg {
    static constexpr int NSTAGE = NT > 64 ? 3 : 4;
    static constexpr int A_ATOM = GM_ROWS * 128, W_ATOM = NT * 128;
    static constexpr int A_STAGE = 2 * A_ATOM, W_STAGE = 2 * W_ATOM;
    static constexpr int OFF_W = NSTAGE * A_STAGE;
    static constexpr int OFF_BAR = OFF_W + NSTAGE * W_STAGE;
    static constexpr int BYTES = OFF_BAR + 2 * NSTAGE * 8 + 1024;
    static_assert(BYTES <= 232448, "exceeds the 227 KB shared-memory limit per CTA");
};

struct alignas(64) ConvTmaParams {
    CUtensorMap maps[FCN_MAX_SEGS];
    fcn_conv_args a;
};

__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap *map, int c0, int c1, int c2,
                                            uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
        "[%0], [%1, {%2, %3, %4}], [%5];\n" ::"r"(dst),
        "l"((uint64_t)map), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
        : "memory");
}

template <int NT>
__global__ void __launch_bounds__(GM_THREADS)
conv_gemm_tma_kernel(const __grid_constant__ ConvTmaParams P) {
    using Cfg = GmCfg<NT>;
    constexpr int NSTAGE = Cfg::NSTAGE;
    const fcn_conv_args &p = P.a;
    extern __shared__ uint8_t smem_dyn[];
    uint8_t *smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
    uint8_t *sA = smem, *sW = smem + Cfg::OFF_W;
    uint64_t *bars = (uint64_t *)(smem + Cfg::OFF_BAR);
    uint64_t *full = bars, *empty = bars + NSTAGE;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // GEMM rows are the flattened (frustum, position) rows of the PADDED activation maps: row r = b*P_m + t.
    // The pad rows between frustums are zero, so kernel taps / the stride-2 sampling need no per-frustum
    // handling (pitch of every source == stride * P_m) and every 128-row tile is fully used.
    const int r0 = blockIdx.x * GM_ROWS;
    const int n_tile = blockIdx.y;
    const int NS = p.K_pad / 64;

    if (tid == 0) {
        for (int i = 0; i < NSTAGE; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], GM_MMA_WARPS);
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();                 // prologue above overlapped the previous layer's tail
    pdl_launch_dependents();

    if (warp == GM_MMA_WARPS) {
        // ================= TMA producer (one lane): A boxes + weight stage =================
        if (lane == 0) {
            const uint8_t *wsrc = (const uint8_t *)p.w_tc + (size_t)n_tile * NS * Cfg::W_STAGE;
            int seg = 0, kbi = 0;                    // running (segment, K block inside the segment)
            for (int s = 0; s < NS; ++s) {
                const int st = s % NSTAGE, ph = (s / NSTAGE) & 1;
                mbar_wait(&empty[st], ph ^ 1);
                mbar_arrive_expect_tx(&full[st], Cfg::A_STAGE + Cfg::W_STAGE);
#pragma unroll
                for (int a = 0; a < 2; ++a) {
                    const uint32_t dst = smem_u32(sA) + st * Cfg::A_STAGE + a * Cfg::A_ATOM;
                    if (seg < p.n_seg) {
                        const fcn_conv_seg &sg = p.seg[seg];
                        tma_load_3d(dst, &P.maps[seg], kbi * 32, r0 * sg.stride + sg.tap, 0, &full[st]);
                        if (++kbi >= ((sg.C + 31) >> 5)) { kbi = 0; ++seg; }
                    } else {   // K padding block: a box fully outside the channel range -> zeros
                        tma_load_3d(dst, &P.maps[0], 1 << 20, 0, 0, &full[st]);
                    }
                }
                bulk_g2s(sW + st * Cfg::W_STAGE, wsrc + (size_t)s * Cfg::W_STAGE, Cfg::W_STAGE, &full[st]);
            }
        }
    } else {
        // ================= consumers: warpgroup wg multiplies rows [64 wg, 64 wg + 64), then stores them =====
        const int wg = warp >> 2;
        float acc[NT / 2];
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
        const uint64_t adesc0 = make_desc_sw128(smem_u32(sA) + wg * (64 * 128));
        const uint64_t bdesc0 = make_desc_sw128(smem_u32(sW));
        int prev = -1;
        for (int s = 0; s < NS; ++s) {
            const int st = s % NSTAGE, ph = (s / NSTAGE) & 1;
            mbar_wait(&full[st], ph);
            const uint64_t ad = adesc0 + (uint64_t)(st * (Cfg::A_STAGE >> 4));
            const uint64_t bd = bdesc0 + (uint64_t)(st * (Cfg::W_STAGE >> 4));
            wgmma_fence();
            fence_acc(acc);
#pragma unroll
            for (int a = 0; a < 2; ++a)
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    wgmma_tf32<NT>(acc, ad + (uint64_t)(a * (Cfg::A_ATOM >> 4) + 2 * k),
                                   bd + (uint64_t)(a * (Cfg::W_ATOM >> 4) + 2 * k), (s | a | k) != 0);
            wgmma_commit();
            fence_acc(acc);
            wgmma_wait<1>();                            // the previous stage's group has retired
            if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
            prev = st;
        }
        wgmma_wait<0>();
        fence_acc(acc);
        conv_store_fragment<NT>(acc, p, r0 + 64 * wg, n_tile * NT);
    }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn == nullptr) {
        void *ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)ptr;
    }
    return fn;
}

template <int NT>
static int launch_gm(const ConvTmaParams &P, cudaStream_t stream) {
    using Cfg = GmCfg<NT>;
    auto kern = conv_gemm_tma_kernel<NT>;
    FCN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::BYTES));
    const fcn_conv_args &a = P.a;
    dim3 grid(ceil_div(a.B * a.P_m, GM_ROWS), a.n_cols / NT);
    static const int prio = env_priority("FCN_PRIO_CONV");
    FCN_CUDA(launch_pdl_prio(prio, kern, grid, dim3(GM_THREADS), (size_t)Cfg::BYTES, stream, P));
    return FCN_OK;
}

// precision 3: N tile 128, precision 4: N tile 64; a.tmaps = host pointer to n_seg 128-byte tensor maps.
int conv_gemm_tma(const fcn_conv_args &a, cudaStream_t stream) {
    FCN_REQUIRE(a.w_tc != nullptr, "NULL tensor-core weight image");
    FCN_REQUIRE(a.tmaps != nullptr, "NULL tensor maps (fcn_encode_activation_map)");
    FCN_REQUIRE(a.Cout % 32 == 0, "tensor-core variant needs Cout % 32 == 0");
    FCN_REQUIRE(a.K_pad % 64 == 0, "tensor-core variant needs K_pad % 64 == 0");
    for (int s = 0; s < a.n_seg; ++s) {
        FCN_REQUIRE(a.seg[s].pitch == a.seg[s].stride * a.P_m, "TMA variant: source pitch must equal stride * P_m");
        FCN_REQUIRE(a.seg[s].tap == 0 || a.seg[s].pitch > a.seg[s].T_src,
                    "TMA variant: kernel taps need zero pad rows between frustums (pitch > T_src)");
    }
    if (a.B * a.T_out == 0) return FCN_OK;
    ConvTmaParams P;
    memcpy(P.maps, a.tmaps, sizeof(CUtensorMap) * a.n_seg);
    P.a = a;
    if (a.precision == 4) return launch_gm<64>(P, stream);
    FCN_REQUIRE(a.n_cols % 128 == 0, "n_cols must be a multiple of 128 for the 128-wide N tile");
    return launch_gm<128>(P, stream);
}

}  // namespace fcn

using namespace fcn;

extern "C" int fcn_encode_activation_map(void *out_map_128B, const float *base, int B, int T, int ld,
                                         int t_stride) {
    FCN_REQUIRE(out_map_128B && base, "NULL pointer");
    FCN_REQUIRE(B >= 1 && T >= 1 && ld >= 4 && ld % 4 == 0, "bad shape");
    FCN_REQUIRE(t_stride == 1 || t_stride == 2, "t_stride must be 1 or 2");
    EncodeTiledFn fn = encode_fn();
    if (fn == nullptr) return fcn::invalid(__func__, "cuTensorMapEncodeTiled is not available in this driver");
    static_assert(sizeof(CUtensorMap) == 128, "CUtensorMap is 128 bytes");
    CUtensorMap m;
    const cuuint64_t gdim[3] = {(cuuint64_t)ld, (cuuint64_t)T, (cuuint64_t)B};
    const cuuint64_t gstr[2] = {(cuuint64_t)ld * 4, (cuuint64_t)T * ld * 4};
    const cuuint32_t box[3] = {32, (cuuint32_t)(GM_ROWS * t_stride), 1};
    const cuuint32_t estr[3] = {1, (cuuint32_t)t_stride, 1};
    CUresult r = fn(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void *)base, gdim, gstr, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        snprintf(fcn::g_err, sizeof(fcn::g_err), "%s: cuTensorMapEncodeTiled failed with CUresult %d", __func__, (int)r);
        return FCN_ERR_CUDA;
    }
    memcpy(out_map_128B, &m, 128);
    return FCN_OK;
}

extern "C" int fcn_encode_store_map(void *out_map_128B, const float *base, int rows, int inner) {
    FCN_REQUIRE(out_map_128B && base, "NULL pointer");
    FCN_REQUIRE(rows >= 1 && inner >= 32 && inner % 4 == 0, "bad shape");
    EncodeTiledFn fn = encode_fn();
    if (fn == nullptr) return fcn::invalid(__func__, "cuTensorMapEncodeTiled is not available in this driver");
    CUtensorMap m;
    const cuuint64_t gdim[3] = {(cuuint64_t)inner, (cuuint64_t)rows, 1};
    const cuuint64_t gstr[2] = {(cuuint64_t)inner * 4, (cuuint64_t)rows * inner * 4};
    const cuuint32_t box[3] = {32, 32, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = fn(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void *)base, gdim, gstr, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        snprintf(fcn::g_err, sizeof(fcn::g_err), "%s: cuTensorMapEncodeTiled failed with CUresult %d", __func__, (int)r);
        return FCN_ERR_CUDA;
    }
    memcpy(out_map_128B, &m, 128);
    return FCN_OK;
}
