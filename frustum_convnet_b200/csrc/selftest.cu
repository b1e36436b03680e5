// Self-test of the wgmma building blocks in isolation (descriptor encodings, swizzled operand
// layouts, accumulator fragment layout): D[128 x N] = A[128 x K] * W[N x K]^T with one warpgroup,
// N in {64, 128, 256} (m64nNk8).  The two 64-row halves run one after the other, so at most 128
// accumulators per thread are live (the N = 256 tile of the persistent FCN kernel).
// A is written to shared memory by threads (as the PointNet epilogues do), W arrives as the
// pre-swizzled stage image produced by the host packer through a bulk copy.
#include "common.cuh"
#include "wgmma.cuh"

namespace fcn {
using namespace gmma;

template <int N>
__global__ void __launch_bounds__(128, 1)
wgmma_selftest_kernel(int K, const float *__restrict__ A, const uint8_t *__restrict__ w_img,
                      float *__restrict__ D) {
    extern __shared__ uint8_t smem_dyn[];
    uint8_t *smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
    const int KB = K / 32;
    uint8_t *sA = smem;                      // KB x [128][128 B]
    uint8_t *sW = sA + KB * 16384;           // KB x [N][128 B]
    uint64_t *bar = (uint64_t *)(sW + KB * N * 128);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        mbar_init(bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    // A: thread = row, rounded to TF32, swizzled
    for (int k = 0; k < K; ++k) {
        const float v = to_tf32(A[(size_t)tid * K + k]);
        *(float *)(sA + (k >> 5) * 16384 + sw128_offset(tid, k & 31)) = v;
    }
    fence_proxy_async();
    if (tid == 0) {
        mbar_arrive_expect_tx(bar, KB * N * 128);
        bulk_g2s(sW, w_img, KB * N * 128, bar);
    }
    __syncthreads();
    mbar_wait(bar, 0);
    for (int h = 0; h < 2; ++h) {
        float acc[N / 2];
#pragma unroll
        for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
        wgmma_fence();
        fence_acc(acc);
        for (int kb = 0; kb < KB; ++kb)
#pragma unroll
            for (int k = 0; k < 4; ++k)
                wgmma_tf32<N>(acc, make_desc_sw128(smem_u32(sA) + kb * 16384 + h * 8192 + k * 32),
                              make_desc_sw128(smem_u32(sW) + kb * N * 128 + k * 32), (kb | k) != 0);
        wgmma_commit();
        wgmma_wait<0>();
        fence_acc(acc);
#pragma unroll
        for (int i = 0; i < N / 2; ++i)
            D[(size_t)(64 * h + frag_row(i, warp, lane)) * N + frag_col(i, lane)] = acc[i];
    }
}

template <int N>
static int launch_selftest(int K, const float *A, const void *w_img, float *D, cudaStream_t stream) {
    const int smem = (K / 32) * (16384 + N * 128) + 8 + 1024;
    FCN_CUDA(cudaFuncSetAttribute(wgmma_selftest_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    wgmma_selftest_kernel<N><<<1, 128, smem, stream>>>(K, A, (const uint8_t *)w_img, D);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

}  // namespace fcn

using namespace fcn;

extern "C" int fcn_selftest_umma(int N, int K, const float *A, const void *w_img, float *D,
                                 fcn_stream_t stream) {
    FCN_REQUIRE(N == 64 || N == 128 || N == 256, "N must be 64, 128 or 256");
    FCN_REQUIRE(K >= 32 && K % 32 == 0, "K must be a positive multiple of 32");
    FCN_REQUIRE((K / 32) * (16384 + N * 128) + 8 + 1024 <= 232448,
                "K too large for shared memory: K <= 256 (N = 64), 224 (N = 128), 128 (N = 256)");
    FCN_REQUIRE(A && w_img && D, "NULL pointer");
    if (N == 64) return launch_selftest<64>(K, A, w_img, D, (cudaStream_t)stream);
    if (N == 128) return launch_selftest<128>(K, A, w_img, D, (cudaStream_t)stream);
    return launch_selftest<256>(K, A, w_img, D, (cudaStream_t)stream);
}
