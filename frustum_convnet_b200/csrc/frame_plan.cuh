// The slot policy of the single-frame entries: fcn_frame_extract (csrc/frame_extract.cu), fcn_frame_refine_extract
// (csrc/frame_refine.cu) and fcn_sunrgbd_frame_extract (csrc/sunrgbd_frame.cu).  Each entry's setup kernel takes
// its frame counts and candidate slots with frame_count and frame_candidate, and its slot kernel runs frame_plan with
// the stage's own slot test and tables.
#pragma once

#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace fcn {

// Frame count c clamped to [0, P]; a count past P sets FCN_FRAME_SCAN_POINTS and a detection count nd past D sets
// FCN_FRAME_DETS.
__device__ __forceinline__ int frame_count(int c, int nd, int P, int D, int &bits) {
    bits |= (c > P ? FCN_FRAME_SCAN_POINTS : 0) | (nd > D ? FCN_FRAME_DETS : 0);
    return c < 0 ? 0 : (c > P ? P : c);
}

// Slot d = f * D + j of frame f: f when it is one of the frame's first det_counts[f] detections, its class is in
// [0, num_classes) with its class_mask bit set and its box is finite, else -1.  A detection of another class or
// with a non-finite box sets FCN_FRAME_BAD_DET.
__device__ __forceinline__ int frame_candidate(int d, int D, int num_classes, unsigned class_mask,
                                               const int32_t *__restrict__ det_counts,
                                               const int32_t *__restrict__ det_class,
                                               const double *__restrict__ boxes, int &bits) {
    const int f = d / D;
    if (d - f * D >= det_counts[f]) return -1;
    const int c = det_class[d];
    const double *b = boxes + 4 * (size_t)d;
    const bool ok = c >= 0 && c < num_classes && isfinite(b[0]) && isfinite(b[1]) && isfinite(b[2]) && isfinite(b[3]);
    if (!ok) bits |= FCN_FRAME_BAD_DET;
    return ok && ((class_mask >> c) & 1u) ? f : -1;
}

// One CTA of THREADS threads over F frames of S slots each (slot d = f * S + j).  One thread per frame walks its
// slots in order: count(d, bits) gives the points slot d would keep, or -1 when it is no frustum, and the slot fits
// while the frame's running point count stays <= Pout (saturating, so the budget drops a suffix; a slot that does
// not fit sets FCN_FRAME_OUT_POINTS).  c2[d] is the kept points of slot d, -1 when dropped.  The classes cls[d] of
// the kept slots are ranked by first appearance, 4 bits a class in one word (15: no rank), into seg_class (NC a
// frame, -1 past the last rank).  Exclusive sums over the frames give kept slot d its batch entry k and output
// position base[d] (written for every slot); the entry's valid, cls_index and seg are written here and the rest by
// kept(k, d, c, base).  Then the B - K dummy entries: each adds one point at p, offsets[k + 1] = p + 1, and zero
// tables, with dummy(k, p) writing the stage's own.
template <int NC, int THREADS, typename Count, typename Kept, typename Dummy>
__device__ __forceinline__ void frame_plan(int F, int S, int Pout, const int32_t *__restrict__ cls,
                                           int32_t *__restrict__ c2, long long *__restrict__ base,
                                           int32_t *__restrict__ seg_class, int32_t *__restrict__ offsets,
                                           int32_t *__restrict__ valid, int32_t *__restrict__ cls_index,
                                           int32_t *__restrict__ seg, int32_t *status, Count count, Kept kept,
                                           Dummy dummy) {
    static_assert(NC >= 1 && NC <= 15, "class ranks take 4 bits a class, 15 meaning none");
    using Scan = cub::BlockScan<int, THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    const int B = F * S;
    int bits = 0, k_run = 0, m_run = 0;
    for (int f0 = 0; f0 < F; f0 += THREADS) {
        const int f = f0 + threadIdx.x;
        unsigned long long rank = ~0ull;
        int k = 0, m = 0;
        if (f < F) {
            int nr = 0, run = 0;
            for (int j = 0; j < S; ++j) {
                const int d = f * S + j;
                int c = count(d, bits);
                if (c >= 0) {
                    run = min(run + c, Pout + 1);
                    if (run > Pout) {
                        bits |= FCN_FRAME_OUT_POINTS;
                        c = -1;
                    }
                }
                c2[d] = c;
                if (c >= 0) {
                    const int cl = cls[d];
                    if (((rank >> (4 * cl)) & 15) == 15) {
                        seg_class[NC * f + nr] = cl;
                        rank &= ~(15ull << (4 * cl));
                        rank |= (unsigned long long)nr++ << (4 * cl);
                    }
                    ++k;
                    m += c;
                }
            }
            for (int q = nr; q < NC; ++q) seg_class[NC * f + q] = -1;
        }
        int kx, kt, mx, mt;
        Scan(tmp).ExclusiveSum(k, kx, kt);
        __syncthreads();
        Scan(tmp).ExclusiveSum(m, mx, mt);
        if (f < F) {
            int kk = k_run + kx;
            long long mm = m_run + mx;
            for (int j = 0; j < S; ++j) {
                const int d = f * S + j, c = c2[d];
                base[d] = mm;
                if (c < 0) continue;
                const int cl = cls[d];
                valid[kk] = 1;
                cls_index[kk] = cl;
                seg[kk] = NC * f + (int)((rank >> (4 * cl)) & 15);
                kept(kk, d, c, mm);
                ++kk;
                mm += c;
            }
        }
        k_run += kt;
        m_run += mt;
        __syncthreads();
    }
    if (threadIdx.x == 0) offsets[0] = 0;
    for (int k = k_run + threadIdx.x; k < B; k += THREADS) {
        const int p = m_run + (k - k_run);
        offsets[k + 1] = p + 1;
        valid[k] = 0;
        cls_index[k] = 0;
        seg[k] = 0;
        dummy(k, p);
    }
    if (bits) atomicOr(status, bits);
}

}  // namespace fcn
