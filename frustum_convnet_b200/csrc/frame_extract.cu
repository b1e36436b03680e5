// The frame kernels of fcn_frame_extract (C ABI section (21), entry in csrc/frustum_extract.cu): section (15)'s count
// and write kernels run over F * D detection slots of fixed capacities, with these around them:
//   frame_setup  clamped per-frame counts, the scan offsets of the packed scans and the candidate slots;
//   frame_pack   the frames' scans packed back to back for the in-image stage;
//   frame_slots  after the count pass: each frame's P_out budget, the batch entry and output position of every kept
//                frustum (what the write kernel is handed), the batch tables and the dummy entries.
#include <cub/block/block_scan.cuh>

#include "common.cuh"
#include "frame_extract.cuh"
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
        int n = 0;
        if (f < F) {
            const int c = a.scan_counts[f], nd = a.det_counts[f];
            n = c < 0 ? 0 : (c > P ? P : c);
            bits |= (c > P ? FCN_FRAME_SCAN_POINTS : 0) | (nd > D ? FCN_FRAME_DETS : 0);
        }
        int off, total;
        Scan(tmp).ExclusiveSum(n, off, total);
        if (f < F) so[f] = run + off;
        run += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) so[F] = run;
    for (int d = threadIdx.x; d < F * D; d += FRAME_THREADS) {
        const int f = d / D, nd = a.det_counts[f];
        int fr = -1;
        if (d - f * D < nd) {
            const int c = a.det_class[d];
            const double *b = a.boxes + 4 * (size_t)d;
            const bool ok = c >= 0 && c < 3 && isfinite(b[0]) && isfinite(b[1]) && isfinite(b[2]) && isfinite(b[3]);
            if (!ok) bits |= FCN_FRAME_BAD_DET;
            else if ((a.class_mask >> c) & 1u) fr = f;
        }
        det_frame[d] = fr;
    }
    if (bits) atomicOr(a.status, bits);
}

// grid (P / FX_THREADS, F): frame f's first n_f scan rows to packed[so[f], so[f + 1])
__global__ void __launch_bounds__(FX_THREADS) frame_pack_kernel(const float4 *__restrict__ scans, int P,
                                                                const int32_t *__restrict__ so,
                                                                float4 *__restrict__ packed) {
    const int f = blockIdx.y, i = blockIdx.x * FX_THREADS + threadIdx.x;
    if (i < so[f + 1] - so[f]) packed[so[f] + i] = scans[(size_t)f * P + i];
}

// One CTA, after the count pass: frame f's kept frustums, in slot order, fit while the frame's kept points up to and
// including theirs are at most P_out; the others are dropped (c2 = -1).  The fitting ones get batch entry k and output
// position base by exclusive sums over all slots, so the write kernel, handed (c2, k, base), stores them compactly
// and no store is cut short.  Then the batch tables of the kept entries and the B - K dummy entries.
__global__ void __launch_bounds__(FRAME_THREADS)
frame_slots_kernel(const fcn_frame_extract_args a, const int32_t *__restrict__ det_points,
                   const long long *__restrict__ cnt_pos, int32_t *__restrict__ c2, int32_t *__restrict__ kpos,
                   long long *__restrict__ base, int32_t *__restrict__ rank) {
    using Scan = cub::BlockScan<int, FRAME_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    const int F = a.num_frames, D = a.det_capacity, B = F * D, Pout = a.out_capacity;
    int bits = 0;
    // class ranks by first appearance among each frame's kept detections that fit its budget (the test of the loop
    // below), so a class whose frustums were all dropped for the budget gets no segment
    for (int f = threadIdx.x; f < F; f += FRAME_THREADS) {
        int r[3] = {-1, -1, -1}, n = 0;
        for (int j = 0; j < D; ++j) {
            const int d = f * D + j;
            if (det_points[d] < 0 || cnt_pos[d] - cnt_pos[(size_t)f * D] + det_points[d] > Pout) continue;
            const int c = a.det_class[d];
            if (r[c] < 0) {
                a.seg_class[3 * f + n] = c;
                r[c] = n++;
            }
        }
        for (int k = n; k < 3; ++k) a.seg_class[3 * f + k] = -1;
        for (int c = 0; c < 3; ++c) rank[3 * f + c] = r[c];
        if (cnt_pos[(size_t)(f + 1) * D] - cnt_pos[(size_t)f * D] > Pout) bits |= FCN_FRAME_OUT_POINTS;
    }
    __syncthreads();
    int k_run = 0, m_run = 0;
    for (int d0 = 0; d0 < B; d0 += FRAME_THREADS) {
        const int d = d0 + threadIdx.x;
        int c = -1;
        if (d < B && det_points[d] >= 0) {
            const int f = d / D;
            const long long end = cnt_pos[d] - cnt_pos[(size_t)f * D] + det_points[d];
            c = end <= Pout ? det_points[d] : -1;
        }
        int kx, kt, mx, mt;
        Scan(tmp).ExclusiveSum(c >= 0 ? 1 : 0, kx, kt);
        __syncthreads();
        Scan(tmp).ExclusiveSum(c >= 0 ? c : 0, mx, mt);
        if (d < B) {
            c2[d] = c;
            kpos[d] = k_run + kx;
            base[d] = m_run + mx;
            if (c >= 0) {
                const int k = k_run + kx, f = d / D, cls = a.det_class[d];
                a.valid[k] = 1;
                a.cls_index[k] = cls;
                a.rgb_prob[k] = a.det_prob[d];
                a.seg[k] = 3 * f + rank[3 * f + cls];
            }
        }
        k_run += kt;
        m_run += mt;
        __syncthreads();
    }
    if (threadIdx.x == 0) a.offsets[0] = 0;
    for (int k = k_run + threadIdx.x; k < B; k += FRAME_THREADS) {
        const int p = m_run + (k - k_run);
        a.offsets[k + 1] = p + 1;
        reinterpret_cast<float4 *>(a.points)[p] = make_float4(0.f, 0.f, 0.f, 0.f);
        a.frustum_angle[k] = 0.0;
        const double bx[4] = {0.0, 0.0, 1.0, 1.0};
        for (int i = 0; i < 4; ++i) a.box2d[4 * (size_t)k + i] = bx[i];
        for (int i = 0; i < 12; ++i) a.P[12 * (size_t)k + i] = (i == 0 || i == 5 || i == 10) ? 1.0 : 0.0;
        a.det_index[k] = -1;
        a.valid[k] = 0;
        a.cls_index[k] = 0;
        a.rgb_prob[k] = 0.f;
        a.seg[k] = 0;
    }
    if (bits) atomicOr(a.status, bits);
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

cudaError_t frame_slots(const fcn_frame_extract_args &a, const int32_t *det_points, const long long *cnt_pos,
                        int32_t *c2, int32_t *kpos, long long *base, int32_t *rank, cudaStream_t s) {
    frame_slots_kernel<<<1, FRAME_THREADS, 0, s>>>(a, det_points, cnt_pos, c2, kpos, base, rank);
    return cudaGetLastError();
}

}  // namespace fcn
