// SUN-RGBD 3-D detection evaluation on the device (C ABI section (14)): eval_det / eval_det_cls of the reference
// (train/sunrgbd_eval/eval_det.py:41-231, ovthresh 0.25 by default, use_07_metric = False) - per class the precision /
// recall curve over the detections in score order and the VOC average precision.
//
// The reference walks the detections of a class in score order and, for each, calls Boost once per ground truth of the
// same image.  Here:
//   fcn_sunrgbd_eval_match   overlap  one thread per detection: the 3-D IoU (rbbox_iou_3d_pair<double>, box_ops.h:
//                                     173-260) against every ground truth of its (class, image) segment in order,
//                                     the first maximum with strict '>', and the candidate ground truth when that
//                                     maximum exceeds ovthresh (:138-152);
//                            sort     stable segmented sort of the scores per class, descending;
//                            claim    one thread per sorted position: atomicMin of the position into the candidate's
//                                     claim slot.  With no fall-back to a second ground truth (:152-157) a detection
//                                     is a TP exactly when it is the best-ranked detection naming its candidate, so
//                                     the sequential walk reduces to that minimum (order-free, deterministic);
//   fcn_sunrgbd_eval_curves  curves   one CTA per class: TP flags, their running sum (tp, fp = rank - tp), rec and
//                                     prec (:162-166), the precision envelope as a suffix maximum and the AP sum of
//                                     voc_ap (:59-71), in a fixed order.
#include <cub/cub.cuh>

#include <cfloat>
#include <cmath>

#include "box_iou.cuh"
#include "common.cuh"

namespace fcn {

constexpr int SE_THREADS = 256;
constexpr int SE_CURVE_THREADS = 512;

// the class of detection d: the last c with det_class_offsets[c] <= d (empty classes skipped)
__device__ __forceinline__ int se_class_of(const int32_t *__restrict__ off, int num_classes, int d) {
    int lo = 0, hi = num_classes - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= d) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(SE_THREADS)
se_overlap_kernel(int num_det, int num_classes, int num_segments, double ovthresh, const double *__restrict__ gt,
                  const double *__restrict__ det, const double *__restrict__ score,
                  const int32_t *__restrict__ det_seg, const int32_t *__restrict__ seg_off,
                  const int32_t *__restrict__ gt_cls_off, const int32_t *__restrict__ det_cls_off,
                  int32_t *__restrict__ cand, double *__restrict__ keys, int32_t *__restrict__ vals,
                  int32_t *__restrict__ status) {
    const int d = blockIdx.x * SE_THREADS + threadIdx.x;
    if (d >= num_det) return;
    keys[d] = score[d] + 0.0;                  // -0.0 -> +0.0: the two zeros tie
    vals[d] = d;
    const int s = det_seg[d];
    int best = -1;
    if (s != -1) {
        const int c = se_class_of(det_cls_off, num_classes, d);
        const int g0 = (s >= 0 && s < num_segments) ? seg_off[s] : -1, g1 = g0 >= 0 ? seg_off[s + 1] : -1;
        if (g0 < gt_cls_off[c] || g1 > gt_cls_off[c + 1]) {
            atomicOr(status + c, FCN_SUNRGBD_BAD_SEGMENT);
        } else {
            const double *bb = det + (size_t)d * 24;
            double ovmax = -INFINITY;
            int jmax = -1;
            for (int j = g0; j < g1; ++j) {
                const double iou = rbbox_iou3d_d(bb, gt + (size_t)j * 24);
                if (iou > ovmax) {
                    ovmax = iou;
                    jmax = j;
                }
            }
            if (ovmax > ovthresh) best = jmax;
        }
    }
    cand[d] = best;
}

__global__ void __launch_bounds__(SE_THREADS)
se_claim_kernel(int num_det, const int32_t *__restrict__ sorted_det, const int32_t *__restrict__ cand,
                int32_t *__restrict__ first) {
    const int p = blockIdx.x * SE_THREADS + threadIdx.x;
    if (p >= num_det) return;
    const int j = cand[sorted_det[p]];
    if (j >= 0) atomicMin(first + j, p);
}

struct SeMax {
    __device__ double operator()(double a, double b) const { return a < b ? b : a; }
};

// One CTA per class.  rec / prec are written in the forward pass and read back by the same CTA in the backward pass
// (after __syncthreads), so they are plain pointers: no read-only cache path.
__global__ void __launch_bounds__(SE_CURVE_THREADS)
se_curves_kernel(const int32_t *__restrict__ gt_cls_off, const int32_t *__restrict__ det_cls_off,
                 const int32_t *__restrict__ sorted_det, const int32_t *__restrict__ cand,
                 const int32_t *__restrict__ first, const int32_t *__restrict__ status, double *rec, double *prec,
                 fcn_sunrgbd_eval_result *__restrict__ out) {
    using ScanI = cub::BlockScan<int, SE_CURVE_THREADS>;
    using ScanD = cub::BlockScan<double, SE_CURVE_THREADS>;
    using Reduce = cub::BlockReduce<double, SE_CURVE_THREADS>;
    __shared__ union {
        typename ScanI::TempStorage si;
        typename ScanD::TempStorage sd;
        typename Reduce::TempStorage r;
    } tmp;
    const int c = blockIdx.x, tid = threadIdx.x;
    const int off = det_cls_off[c], nd = det_cls_off[c + 1] - off;
    const int npos = gt_cls_off[c + 1] - gt_cls_off[c];
    const double dnpos = (double)npos;
    // forward: tp = running count of TP flags; fp = rank - tp
    int carry = 0;
    for (int base = 0; base < nd; base += SE_CURVE_THREADS) {
        const int k = base + tid;
        int flag = 0;
        if (k < nd) {
            const int j = cand[sorted_det[off + k]];
            flag = j >= 0 && first[j] == off + k;
        }
        int incl, total;
        ScanI(tmp.si).InclusiveSum(flag, incl, total);
        if (k < nd) {
            const int tp = carry + incl, fp = k + 1 - tp;
            rec[off + k] = (double)tp / dnpos;
            prec[off + k] = (double)tp / fmax((double)tp + (double)fp, DBL_EPSILON);
        }
        carry += total;
        __syncthreads();
    }
    // backward (chunks of SE_CURVE_THREADS positions from the end): envelope mpre[k + 1] = max(prec[k..nd-1], 0) and the terms (rec[k] - rec[k-1]) * mpre[k + 1] where the
    // recall changes; the last term (1 - rec[nd-1]) * 0 belongs to thread 0
    double acc = 0.0;
    if (tid == 0) {
        const double last = nd > 0 ? rec[off + nd - 1] : 0.0;
        if (1.0 != last) acc = (1.0 - last) * 0.0;
    }
    double env = 0.0;
    for (int end = nd; end > 0; end -= SE_CURVE_THREADS) {
        const int k = end - 1 - tid;
        const double p = k >= 0 ? prec[off + k] : 0.0;
        double m, chunk_max;
        ScanD(tmp.sd).InclusiveScan(p, m, SeMax(), chunk_max);
        m = env < m ? m : env;
        if (k >= 0) {
            const double r = rec[off + k], r0 = k > 0 ? rec[off + k - 1] : 0.0;
            if (r != r0) acc = __dadd_rn(acc, __dmul_rn(r - r0, m));   // no contraction: rounded products
        }
        env = env < chunk_max ? chunk_max : env;
        __syncthreads();
    }
    const double ap = Reduce(tmp.r).Sum(acc);
    if (tid == 0) {
        out[c].ap = ap;
        out[c].npos = npos;
        out[c].nd = nd;
        out[c].status = status[c];
        out[c].reserved = 0;
    }
}

// ------------------------------------------------------------------------------------------------ host side
struct SeWs {
    int32_t *cand, *vals, *sorted_det, *first, *status;
    double *keys, *sorted_keys;
    void *temp;
    size_t temp_bytes;
};

static cudaError_t se_layout(const fcn_sunrgbd_eval_args *a, Carve &c, SeWs &w) {
    const size_t D = (size_t)a->num_det, G = (size_t)a->num_gt, C = (size_t)a->num_classes;
    w.temp_bytes = 0;
    if (a->num_det > 0) {
        cudaError_t e = cub::DeviceSegmentedSort::StableSortPairsDescending(
            nullptr, w.temp_bytes, (const double *)nullptr, (double *)nullptr, (const int32_t *)nullptr,
            (int32_t *)nullptr, a->num_det, a->num_classes, (const int32_t *)nullptr, (const int32_t *)nullptr);
        if (e != cudaSuccess) return e;
    }
    w.cand = (int32_t *)c.take(D * 4);
    w.vals = (int32_t *)c.take(D * 4);
    w.sorted_det = (int32_t *)c.take(D * 4);
    w.keys = (double *)c.take(D * 8);
    w.sorted_keys = (double *)c.take(D * 8);
    w.first = (int32_t *)c.take(G * 4);
    w.status = (int32_t *)c.take(C * 4);
    w.temp = c.take(w.temp_bytes);
    return cudaSuccess;
}

// Host-side checks shared by every entry: counts, pointers and the host copies of the offsets.
static int se_check(const fcn_sunrgbd_eval_args *a, const char *fn) {
    if (a == nullptr) return invalid(fn, "NULL args");
    if (a->num_classes < 0 || a->num_gt < 0 || a->num_gt_segments < 0 || a->num_det < 0)
        return invalid(fn, "negative count (num_classes, num_gt, num_gt_segments, num_det must be >= 0)");
    if (a->num_classes > FCN_SUNRGBD_MAX_CLASSES || a->num_gt > (1 << 28) || a->num_det > (1 << 28) ||
        a->num_gt_segments > a->num_gt)
        return invalid(fn, "too many records (num_classes <= FCN_SUNRGBD_MAX_CLASSES, num_gt and num_det <= 2^28, "
                           "num_gt_segments <= num_gt)");
    if (!a->host_gt_segment_offsets || !a->host_gt_class_offsets || !a->host_det_class_offsets)
        return invalid(fn, "NULL host offsets");
    if (!a->gt_segment_offsets || !a->gt_class_offsets || !a->det_class_offsets || (a->num_gt > 0 && !a->gt_corners) ||
        (a->num_det > 0 && (!a->det_corners || !a->det_scores || !a->det_segments)))
        return invalid(fn, "NULL pointer");
    const int32_t *so = a->host_gt_segment_offsets, *gc = a->host_gt_class_offsets, *dc = a->host_det_class_offsets;
    if (!offsets_ok(so, a->num_gt_segments, a->num_gt) || !offsets_ok(gc, a->num_classes, a->num_gt) ||
        !offsets_ok(dc, a->num_classes, a->num_det))
        return invalid(fn, "offsets must start at 0, never decrease and end at num_gt / num_det");
    for (int c = 0, s = 0; c <= a->num_classes; ++c) {          // every class boundary is a segment boundary
        while (s < a->num_gt_segments && so[s] < gc[c]) ++s;
        if (so[s] != gc[c]) return invalid(fn, "a ground-truth segment crosses a class boundary");
    }
    return FCN_OK;
}

static int se_prepare(const fcn_sunrgbd_eval_args *a, const char *fn, SeWs &w) {
    const int st = se_check(a, fn);
    if (st != FCN_OK) return st;
    if (!a->workspace || !a->result || (a->num_det > 0 && (!a->rec || !a->prec)))
        return invalid(fn, "NULL workspace or output");
    return carve_workspace(fn, "sunrgbd_eval", a->workspace, a->workspace_bytes,
                           [&](Carve &c) { return se_layout(a, c, w); });
}

}  // namespace fcn

using namespace fcn;

extern "C" long long fcn_sunrgbd_eval_workspace_bytes(const fcn_sunrgbd_eval_args *a) {
    if (se_check(a, __func__) != FCN_OK) return -1;
    SeWs w;
    return workspace_size(__func__, [&](Carve &c) { return se_layout(a, c, w); });
}

extern "C" int fcn_sunrgbd_eval_match(const fcn_sunrgbd_eval_args *a, fcn_stream_t stream) {
    SeWs w;
    const int st = se_prepare(a, __func__, w);
    if (st != FCN_OK) return st;
    cudaStream_t s = (cudaStream_t)stream;
    const int D = a->num_det;
    if (a->num_classes > 0) FCN_CUDA(cudaMemsetAsync(w.status, 0, (size_t)a->num_classes * 4, s));
    if (a->num_gt > 0) FCN_CUDA(cudaMemsetAsync(w.first, 0x7f, (size_t)a->num_gt * 4, s));   // 0x7f7f7f7f: unclaimed
    if (D == 0) return FCN_OK;
    se_overlap_kernel<<<ceil_div(D, SE_THREADS), SE_THREADS, 0, s>>>(
        D, a->num_classes, a->num_gt_segments, a->ovthresh, a->gt_corners, a->det_corners, a->det_scores,
        a->det_segments, a->gt_segment_offsets, a->gt_class_offsets, a->det_class_offsets, w.cand, w.keys, w.vals,
        w.status);
    FCN_LAUNCH_CHECK();
    FCN_CUDA(cub::DeviceSegmentedSort::StableSortPairsDescending(w.temp, w.temp_bytes, w.keys, w.sorted_keys, w.vals,
                                                                 w.sorted_det, D, a->num_classes,
                                                                 a->det_class_offsets, a->det_class_offsets + 1, s));
    se_claim_kernel<<<ceil_div(D, SE_THREADS), SE_THREADS, 0, s>>>(D, w.sorted_det, w.cand, w.first);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

extern "C" int fcn_sunrgbd_eval_curves(const fcn_sunrgbd_eval_args *a, fcn_stream_t stream) {
    SeWs w;
    const int st = se_prepare(a, __func__, w);
    if (st != FCN_OK) return st;
    if (a->num_classes == 0) return FCN_OK;
    se_curves_kernel<<<a->num_classes, SE_CURVE_THREADS, 0, (cudaStream_t)stream>>>(
        a->gt_class_offsets, a->det_class_offsets, w.sorted_det, w.cand, w.first, w.status, a->rec, a->prec,
        a->result);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}
