// Fused detection losses + their gradient w.r.t. the head logits (SURVEY.md 8(f)-2, train half).
//
// Replaces the ~300 PyTorch elementwise / gather / reduction ops of the reference's train branch
// (/root/reference/models/det_base.py:414-503: fg selection, focal loss models/common.py:217-232, Huber losses
// models/model_util.py:9-19, box coding models/box_transform.py:5-65, corner loss models/model_util.py:48-72 +
// det_base.py:449-461, accuracies utils/utils.py:28-50, IoU metrics det_base.py:488-500) AND their autograd backward
// by three tiny launches:
//   det_loss_count_kernel : nfg = #(label == 1), nkeep = #(label != -1)
//   det_loss_rows_kernel  : one thread per (frustum, position) row: every loss term of the row, its hand-derived
//                           gradient w.r.t. the 2 + (3 + 2*NH + 4*NS) logits of the row (scaled by 1/nfg and the
//                           loss weights), accuracies, rotated IoU of the predicted box (box_iou.cuh);
//                           block reduction -> fp32 atomics into 16 accumulators
//   det_loss_final_kernel : the eight losses (det_base.py:505-514) and six metrics (:516-523)
// Means over the foreground rows are sum(w * term) / nfg, exactly the reference's `nonzero()` row selection
// (tests/test_train_host_cpu.py proves the weighted form equal to the selected form incl. gradients).
#include "loss_terms.cuh"

namespace fcn {

__global__ void det_loss_count_kernel(int N, const long long *__restrict__ lab, float *__restrict__ counts) {
    __shared__ int s[2];
    if (threadIdx.x < 2) s[threadIdx.x] = 0;
    __syncthreads();
    int fg = 0, keep = 0;
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < N; r += gridDim.x * blockDim.x) {
        const long long l = lab[r];
        fg += l == 1;
        keep += l != -1;
    }
    atomicAdd(&s[0], fg);
    atomicAdd(&s[1], keep);
    __syncthreads();
    if (threadIdx.x == 0) { atomicAdd(&counts[0], (float)s[0]); atomicAdd(&counts[1], (float)s[1]); }
}

__global__ void __launch_bounds__(128)
det_loss_rows_kernel(const __grid_constant__ fcn_loss_args a, const float *__restrict__ counts, float *__restrict__ acc) {
    __shared__ float s_acc[A_N];
    if (threadIdx.x < A_N) s_acc[threadIdx.x] = 0.f;
    __syncthreads();
    const int N = a.B * a.T2, NH = a.NH, NS = a.NS, W = 3 + 2 * NH + 4 * NS;
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    float v[A_N];
#pragma unroll
    for (int i = 0; i < A_N; ++i) v[i] = 0.f;
#include "loss_row.cuh"
#pragma unroll
    for (int i = 0; i < A_N; ++i) {
        float x = v[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
        if ((threadIdx.x & 31) == 0 && x != 0.f) atomicAdd(&s_acc[i], x);
    }
    __syncthreads();
    if (threadIdx.x < A_N && s_acc[threadIdx.x] != 0.f) atomicAdd(&acc[threadIdx.x], s_acc[threadIdx.x]);
}

// Deterministic mode (fcn_det_loss_deterministic): the same rows; each warp's sums (a fixed butterfly) are added in
// warp order and the CTA's 13 sums go to its slot [CTA][A_N] with plain stores.  dcls / dreg are those of
// det_loss_rows_kernel: they never read the sums.
__global__ void __launch_bounds__(128)
det_loss_rows_det_kernel(const __grid_constant__ fcn_loss_args a, const float *__restrict__ counts,
                         float *__restrict__ slots) {
    __shared__ float s_w[4][A_N];
    const int N = a.B * a.T2, NH = a.NH, NS = a.NS, W = 3 + 2 * NH + 4 * NS;
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    float v[A_N];
#pragma unroll
    for (int i = 0; i < A_N; ++i) v[i] = 0.f;
#include "loss_row.cuh"
#pragma unroll
    for (int i = 0; i < A_N; ++i) {
        float x = v[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
        if ((threadIdx.x & 31) == 0) s_w[threadIdx.x / 32][i] = x;
    }
    __syncthreads();
    if (threadIdx.x < A_N)
        slots[(size_t)blockIdx.x * A_N + threadIdx.x] =
            ((s_w[0][threadIdx.x] + s_w[1][threadIdx.x]) + s_w[2][threadIdx.x]) + s_w[3][threadIdx.x];
}

// acc[i] = the sum of the CTA slots in CTA order (fp64, rounded once)
__global__ void det_loss_slots_kernel(int nblk, const float *__restrict__ slots, float *__restrict__ acc) {
    if (threadIdx.x >= A_N) return;
    double t = 0.0;
    for (int b = 0; b < nblk; ++b) t += (double)slots[(size_t)b * A_N + threadIdx.x];
    acc[threadIdx.x] = (float)t;
}

// out[0..13] = the 14 values of loss_final_values (loss_terms.cuh); out[14..15] = #foreground, #non-ignored rows
__global__ void det_loss_final_kernel(const __grid_constant__ fcn_loss_args a, const float *__restrict__ counts,
                                      const float *__restrict__ acc, float *__restrict__ out) {
    if (threadIdx.x != 0) return;
    loss_final_values(a, acc, counts[0], counts[1], out);
    out[14] = counts[0];
    out[15] = counts[1];
}

}  // namespace fcn

using namespace fcn;

extern "C" int fcn_det_loss(const fcn_loss_args *args, fcn_stream_t stream) {
    FCN_REQUIRE(args != nullptr, "args is NULL");
    const fcn_loss_args &a = *args;
    FCN_REQUIRE(a.B >= 1 && a.T2 >= 1 && a.NH >= 1 && a.NH <= LOSS_MAX_BINS && a.NS >= 1 && a.NS <= LOSS_MAX_BINS, "bad sizes");
    FCN_REQUIRE(a.cls && a.reg && a.center_ref2 && a.cls_label && a.box3d_center && a.box3d_heading && a.box3d_size &&
                    a.size_class && a.mean_size && a.dcls && a.dreg && a.out && a.scratch, "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int N = a.B * a.T2;
    float *counts = a.scratch, *acc = a.scratch + 2;
    FCN_CUDA(cudaMemsetAsync(a.scratch, 0, sizeof(float) * (2 + A_N), st));
    det_loss_count_kernel<<<min(ceil_div(N, 256), 64), 256, 0, st>>>(N, (const long long *)a.cls_label, counts);
    FCN_LAUNCH_CHECK();
    det_loss_rows_kernel<<<ceil_div(N, 128), 128, 0, st>>>(a, counts, acc);
    FCN_LAUNCH_CHECK();
    det_loss_final_kernel<<<1, 32, 0, st>>>(a, counts, acc, a.out);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

// Deterministic variant: slots of the row CTAs after the 16 floats of fcn_det_loss's scratch.  The counts are sums of
// integers: the per-CTA int atomics are exact, and the float atomics over CTAs add integers exactly while the total
// stays below 2^24, which the row bound below guarantees.
static int det_loss_rows_ok(long long rows) { return rows >= 1 && rows <= (1 << 24); }

extern "C" long long fcn_det_loss_deterministic_scratch_floats(long long rows) {
    if (!det_loss_rows_ok(rows)) return 0;
    return 16 + (long long)ceil_div((int)rows, 128) * A_N;
}

extern "C" int fcn_det_loss_deterministic(const fcn_loss_args *args, fcn_stream_t stream) {
    FCN_REQUIRE(args != nullptr, "args is NULL");
    const fcn_loss_args &a = *args;
    FCN_REQUIRE(a.B >= 1 && a.T2 >= 1 && a.NH >= 1 && a.NH <= LOSS_MAX_BINS && a.NS >= 1 && a.NS <= LOSS_MAX_BINS, "bad sizes");
    FCN_REQUIRE(a.cls && a.reg && a.center_ref2 && a.cls_label && a.box3d_center && a.box3d_heading && a.box3d_size &&
                    a.size_class && a.mean_size && a.dcls && a.dreg && a.out && a.scratch, "NULL pointer");
    FCN_REQUIRE(det_loss_rows_ok((long long)a.B * a.T2), "more than 2^24 rows: the float row counts would not be exact");
    cudaStream_t st = (cudaStream_t)stream;
    const int N = a.B * a.T2, nblk = ceil_div(N, 128);
    float *counts = a.scratch, *acc = a.scratch + 2, *slots = a.scratch + 16;
    FCN_CUDA(cudaMemsetAsync(a.scratch, 0, sizeof(float) * 2, st));
    det_loss_count_kernel<<<min(ceil_div(N, 256), 64), 256, 0, st>>>(N, (const long long *)a.cls_label, counts);
    FCN_LAUNCH_CHECK();
    det_loss_rows_det_kernel<<<nblk, 128, 0, st>>>(a, counts, slots);
    FCN_LAUNCH_CHECK();
    det_loss_slots_kernel<<<1, 32, 0, st>>>(nblk, slots, acc);
    FCN_LAUNCH_CHECK();
    det_loss_final_kernel<<<1, 32, 0, st>>>(a, counts, acc, a.out);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}
