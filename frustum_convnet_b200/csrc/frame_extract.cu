// The frame kernels of fcn_frame_extract (C ABI section (21), entry in csrc/frustum_extract.cu): section (15)'s count
// and write kernels run over F * D detection slots of fixed capacities, with these around them:
//   frame_setup  clamped per-frame counts, the scan offsets of the packed scans and the candidate slots;
//   frame_pack   the frames' scans packed back to back for the in-image stage;
//   frame_slots  after the count pass: each frame's P_out budget, the batch entry and output position of every kept
//                frustum (what the write kernel is handed), the batch tables and the dummy entries (frame_plan).
#include <cub/block/block_scan.cuh>

#include "common.cuh"
#include "frame_extract.cuh"
#include "frame_plan.cuh"
#include "frustum_fov.cuh"

namespace fcn {

constexpr int FRAME_THREADS = 1024;

// One CTA: frame f holds n_f = min(scan_counts[f], P) points at so[f] of the packed scans and its first
// min(det_counts[f], D) slots are detections; a slot is a candidate (det_frame = f) when its class is wanted and its
// box finite, else det_frame = -1 (section (15)'s count pass drops it).
__global__ void __launch_bounds__(FRAME_THREADS) frame_setup_kernel(const fcn_frame_extract_args a, int32_t *so,
                                                                    int32_t *det_frame) {
    using Scan = cub::BlockScan<int, FRAME_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    const int F = a.num_frames, P = a.scan_capacity, D = a.det_capacity;
    int run = 0, bits = 0;
    for (int f0 = 0; f0 < F; f0 += FRAME_THREADS) {
        const int f = f0 + threadIdx.x;
        const int n = f < F ? frame_count(a.scan_counts[f], a.det_counts[f], P, D, bits) : 0;
        int off, total;
        Scan(tmp).ExclusiveSum(n, off, total);
        if (f < F) so[f] = run + off;
        run += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) so[F] = run;
    for (int d = threadIdx.x; d < F * D; d += FRAME_THREADS)
        det_frame[d] = frame_candidate(d, D, 3, a.class_mask, a.det_counts, a.det_class, a.boxes, bits);
    if (bits) atomicOr(a.status, bits);
}

// grid (P / FX_THREADS, F): frame f's first n_f scan rows to packed[so[f], so[f + 1])
__global__ void __launch_bounds__(FX_THREADS) frame_pack_kernel(const float4 *__restrict__ scans, int P,
                                                                const int32_t *__restrict__ so,
                                                                float4 *__restrict__ packed) {
    const int f = blockIdx.y, i = blockIdx.x * FX_THREADS + threadIdx.x;
    if (i < so[f + 1] - so[f]) packed[so[f] + i] = scans[(size_t)f * P + i];
}

// One CTA, after the count pass: frame_plan over the F frames of D detection slots, each slot's points from the count
// pass.  The write kernel, handed (c2, kpos, base), stores the kept frustums compactly and reads kpos of those only.
__global__ void __launch_bounds__(FRAME_THREADS)
frame_slots_kernel(const fcn_frame_extract_args a, const int32_t *__restrict__ det_points, int32_t *__restrict__ c2,
                   int32_t *__restrict__ kpos, long long *__restrict__ base) {
    frame_plan<3, FRAME_THREADS>(
        a.num_frames, a.det_capacity, a.out_capacity, a.det_class, c2, base, a.seg_class, a.offsets, a.valid,
        a.cls_index, a.seg, a.status, [&](int d, int &) { return det_points[d]; },
        [&](int k, int d, int, long long) {
            kpos[d] = k;
            a.rgb_prob[k] = a.det_prob[d];
        },
        [&](int k, int p) {
            reinterpret_cast<float4 *>(a.points)[p] = make_float4(0.f, 0.f, 0.f, 0.f);
            a.frustum_angle[k] = 0.0;
            const double bx[4] = {0.0, 0.0, 1.0, 1.0};
            for (int i = 0; i < 4; ++i) a.box2d[4 * (size_t)k + i] = bx[i];
            for (int i = 0; i < 12; ++i) a.P[12 * (size_t)k + i] = (i == 0 || i == 5 || i == 10) ? 1.0 : 0.0;
            a.det_index[k] = -1;
            a.rgb_prob[k] = 0.f;
        });
}

cudaError_t frame_setup(const fcn_frame_extract_args &a, int32_t *so, int32_t *det_frame, float4 *packed,
                        cudaStream_t s) {
    frame_setup_kernel<<<1, FRAME_THREADS, 0, s>>>(a, so, det_frame);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    frame_pack_kernel<<<dim3(ceil_div(a.scan_capacity, FX_THREADS), a.num_frames), FX_THREADS, 0, s>>>(
        (const float4 *)a.scans, a.scan_capacity, so, packed);
    return cudaGetLastError();
}

cudaError_t frame_slots(const fcn_frame_extract_args &a, const int32_t *det_points, int32_t *c2, int32_t *kpos,
                        long long *base, cudaStream_t s) {
    frame_slots_kernel<<<1, FRAME_THREADS, 0, s>>>(a, det_points, c2, kpos, base);
    return cudaGetLastError();
}

}  // namespace fcn
