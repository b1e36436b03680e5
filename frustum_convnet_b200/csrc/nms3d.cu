// Rotated 3-D NMS on the device (SURVEY.md 8(f)-4): replaces the post-processing of test_net_det.py:126-152 ->
// ops/pybind11/rbbox_iou.py:294-311 `rotate_nms_3d_cc` (= the driver's `cube_nms`) -> nms_cpu.h:148-240
// `rotate_non_max_suppression_3d_cpu`, which today costs a device->host copy of every prediction, a Python loop
// per image / class and a CPU Boost polygon clip per box pair.
//
// One CTA per segment (= one image x class list of detections, <= NMS_MAX_DETS boxes; nms.py refuses longer lists,
// the kernel would consider only their first NMS_MAX_DETS rows):
//   1. corners of every box (boxes3d2corners, rbbox_iou.py:121-148) and its axis-aligned bounding cube;
//   2. rank by descending score (the reference: scores.argsort()[::-1]; ties: larger index first, i.e. the
//      reverse of a stable ascending sort, where NaN sorts above every number and -0.0 equals +0.0);
//   3. suppression bit matrix in RANK order: bit (i, j) for j > i is set iff the bounding cubes overlap
//      (standup IoU > 0, nms_cpu.h:192) and the rotated 3-D IoU (box_iou.cuh, the same function as the train
//      metric, incl. its degenerate-ring rule) is >= thresh (nms_cpu.h:226-227);
//   4. greedy scan in rank order by one warp (keep i unless suppressed, then OR row i into the suppressed set);
//   5. the first top_k kept indices (rbbox_iou.py:311 `keep[:top_k]`) in rank order, count per segment.
#include "box_corners.cuh"
#include "box_iou.cuh"
#include "common.cuh"

namespace fcn {

constexpr int NMS_MAX_DETS = 512;
constexpr int NMS_WORDS = NMS_MAX_DETS / 32;
constexpr int NMS_THREADS = 256;

// Row j ranks before row i.  A strict total order, so the ranks are a permutation whatever the scores: NaN above
// every number (numpy sorts NaN last, the reversed order puts it first), equal scores (NaN with NaN, -0.0 with
// +0.0) by the larger index first.
__device__ __forceinline__ bool nms_ranks_before(float sj, int j, float si, int i) {
    const bool nj = sj != sj, ni = si != si;
    if (nj || ni) return nj && (!ni || j > i);
    return sj > si || (sj == si && j > i);
}

__global__ void __launch_bounds__(NMS_THREADS)
nms3d_kernel(const float *__restrict__ dets, const int *__restrict__ seg_offsets, float thresh, int top_k,
             int *__restrict__ keep, int *__restrict__ keep_count, int keep_stride) {
    extern __shared__ unsigned char nms_smem[];
    float *corners = (float *)nms_smem;                              // [n][24], in RANK order
    float *cube = corners + NMS_MAX_DETS * 24;                       // [n][6] min xyz, max xyz
    int *order = (int *)(cube + NMS_MAX_DETS * 6);                   // rank -> original index (inside the segment)
    unsigned *mask = (unsigned *)(order + NMS_MAX_DETS);             // [n][NMS_WORDS]
    const int seg = blockIdx.x;
    const int base = seg_offsets[seg], n = min(seg_offsets[seg + 1] - base, NMS_MAX_DETS);
    const int tid = threadIdx.x;
    const float *d = dets + (size_t)base * 8;
    // ---- rank by descending score (ties: larger index first; NaN first)
    for (int i = tid; i < n; i += NMS_THREADS) {
        const float si = d[i * 8 + 7];
        int rank = 0;
        for (int j = 0; j < n; ++j) {
            const float sj = d[j * 8 + 7];
            rank += nms_ranks_before(sj, j, si, i) ? 1 : 0;
        }
        order[rank] = i;
    }
    __syncthreads();
    for (int r = tid; r < n; r += NMS_THREADS) {
        float c[24];
        box_to_corners(d + (size_t)order[r] * 8, c);
        float mn[3] = {c[0], c[1], c[2]}, mx[3] = {c[0], c[1], c[2]};
#pragma unroll
        for (int i = 0; i < 8; ++i) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                corners[r * 24 + 3 * i + k] = c[3 * i + k];
                mn[k] = fminf(mn[k], c[3 * i + k]);
                mx[k] = fmaxf(mx[k], c[3 * i + k]);
            }
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) { cube[r * 6 + k] = mn[k]; cube[r * 6 + 3 + k] = mx[k]; }
    }
    for (int i = tid; i < n * NMS_WORDS; i += NMS_THREADS) mask[i] = 0u;
    __syncthreads();
    // ---- suppression bits for all pairs i < j (rank order)
    const int npairs = n * (n - 1) / 2;
    for (int p = tid; p < npairs; p += NMS_THREADS) {
        // p -> (i, j), i < j: row i holds n-1-i pairs
        int i = 0, rem = p;
        while (rem >= n - 1 - i) { rem -= n - 1 - i; ++i; }
        const int j = i + 1 + rem;
        const float *a = cube + i * 6, *b = cube + j * 6;
        if (!cubes_overlap(a, b)) continue;      // standup IoU > 0 (rbbox_iou.py:62-96)
        float iou[2];
        rbbox_iou_pair(corners + i * 24, corners + j * 24, iou);
        if (iou[1] >= thresh) atomicOr(&mask[i * NMS_WORDS + (j >> 5)], 1u << (j & 31));
    }
    __syncthreads();
    // ---- greedy scan (one warp: lane = word of the suppressed set)
    if (tid < 32) {
        unsigned supp = 0u;                       // lane w holds word w of the suppressed bit set (n <= 512: 16 words)
        int kept = 0;
        for (int i = 0; i < n; ++i) {
            const unsigned word = __shfl_sync(0xffffffffu, supp, i >> 5);
            if ((word >> (i & 31)) & 1u) continue;
            if (kept < top_k && tid == 0) keep[(size_t)seg * keep_stride + kept] = base + order[i];
            ++kept;
            if (tid < NMS_WORDS) supp |= mask[i * NMS_WORDS + tid];
        }
        if (tid == 0) keep_count[seg] = min(kept, top_k);
    }
}

}  // namespace fcn

using namespace fcn;

extern "C" int fcn_rotate_nms_3d(int num_segments, const float *dets, const int32_t *seg_offsets, float thresh,
                                 int top_k, int32_t *keep, int32_t *keep_count, int keep_stride, fcn_stream_t stream) {
    FCN_REQUIRE(num_segments >= 0 && top_k >= 1 && keep_stride >= 1, "bad sizes");
    if (num_segments == 0) return FCN_OK;
    FCN_REQUIRE(dets && seg_offsets && keep && keep_count, "NULL pointer");
    const size_t smem = (size_t)NMS_MAX_DETS * (24 + 6) * 4 + NMS_MAX_DETS * 4 + (size_t)NMS_MAX_DETS * NMS_WORDS * 4;
    FCN_CUDA(cudaFuncSetAttribute(nms3d_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    nms3d_kernel<<<num_segments, NMS_THREADS, smem, (cudaStream_t)stream>>>(dets, seg_offsets, thresh, top_k, keep,
                                                                            keep_count, keep_stride);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

extern "C" int fcn_rotate_nms_3d_max_dets(void) { return NMS_MAX_DETS; }
