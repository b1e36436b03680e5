// KITTI object evaluation on the device (C ABI section (13)): the offline evaluator of the reference
// (train/kitti_eval/evaluate_object_3d_offline.cpp:56-916) with its semantics unchanged - image 2-D AP with AOS,
// bird's-eye-view (ground) AP and 3-D AP for car, pedestrian and cyclist at the easy, moderate and hard levels,
// as the 41-point precision / AOS vectors and the printed AP.
//
// The evaluator's unit of work is an "evaluation" e = (metric m, class c, difficulty d), 27 of them.  The
// reference recomputes every overlap inside every threshold loop; here each is computed once:
//   fcn_kitti_eval_overlaps    flags   run-level flags from the detections (loadDetections, :157-172);
//                              offsets per image nd_i * ng_i pair slots and ceil(nd_i / 32) mask words (scans);
//                              pairs   one thread per (detection, ground truth) pair and metric: the IoU
//                                      (criterion -1, :229-263, :296-346), or criterion 0 (overlap / detection
//                                      area or volume) when the ground truth is DontCare (:582);
//   fcn_kitti_eval_thresholds  pass 1  one thread per (evaluation, image): cleanData (:383-456) and
//                                      computeStatistics(compute_fp = false) (:458-556) write the TP scores of the
//                                      image into its slots of the evaluation's score segment (-inf elsewhere);
//                              sort    segmented radix sort of the 27 score segments, descending;
//                              recall  one thread per evaluation: getThresholds (:348-381), sequentially;
//   fcn_kitti_eval_statistics  pass 2  one thread per (evaluation, threshold, image): computeStatistics(compute_fp
//                                      = true) with the ignored-detection reassignment (:515-525), the DontCare
//                                      subtraction (:569-591) and, for the image metric, the AOS sum (:594-613);
//                                      each CTA sums its 128 images in a fixed tree into one partial;
//                              final   one thread per evaluation sums the partials in CTA order, then precision,
//                                      AOS and their suffix maximum (:680-699) and the printed AP (:716-720).
// Every sum has a fixed order, so results are bit-identical from run to run and across streams.
//
// The per-thread `assigned_detection` vector of computeStatistics is a bit set in the workspace: one word range per
// (evaluation[, threshold], image), owned by one thread and cleared by it first.
//
// Products that the reference evaluates as separate double operations (x86-64 without FMA) are written with
// __dmul_rn / __dadd_rn so that nvcc does not contract them into fused multiply-adds.
#include <cub/cub.cuh>

#include <cmath>
#include <vector>

#include "box_iou.cuh"
#include "common.cuh"

namespace fcn {

constexpr int KE_THREADS = 128;
constexpr int KE_EVALS = 27;                // metric x class x difficulty
constexpr int KE_PTS = FCN_KITTI_PTS;       // 41 recall steps
constexpr double KE_NO_DETECTION = -10000000;

static_assert(FCN_KITTI_GT_COLS == 15 && FCN_KITTI_DET_COLS == 14, "record layouts");

// ground-truth record columns (the label_2 line with the type replaced by its code)
enum { G_CODE, G_TRUNC, G_OCCL, G_ALPHA, G_X1, G_Y1, G_X2, G_Y2, G_H, G_W, G_L, G_T1, G_T2, G_T3, G_RY };
// detection record columns (the result line without the two unused fields)
enum { D_CODE, D_ALPHA, D_X1, D_Y1, D_X2, D_Y2, D_H, D_W, D_L, D_T1, D_T2, D_T3, D_RY, D_SCORE };

__constant__ int c_min_height[3] = {40, 25, 25};
__constant__ int c_max_occlusion[3] = {0, 1, 2};
__constant__ double c_max_truncation[3] = {0.15, 0.3, 0.5};
__constant__ double c_min_overlap[3][3] = {{0.7, 0.5, 0.5}, {0.7, 0.5, 0.5}, {0.7, 0.5, 0.5}};

// flags[] in the workspace
enum { F_IMAGE = 0, F_GROUND = 3, F_3D = 6, F_NO_AOS = 9, F_COUNT = 16 };

// ------------------------------------------------------------------------------------------------ overlaps
// toPolygon (:271-293): rotation [[c, s], [-s, c]] applied to (+-l/2, +-w/2), then + (t1, t3); clockwise for
// positive l, w.  ublas' prod sums the two products of a row left to right.
__device__ void ke_polygon(const double *r, int ry, int l, int w, int t1, int t3, Pt2d *P) {
    const double c = cos(r[ry]), s = sin(r[ry]);
    const double hl = r[l] / 2, hw = r[w] / 2;
    const double dx[4] = {hl, hl, -hl, -hl}, dz[4] = {hw, -hw, -hw, hw};
    for (int i = 0; i < 4; ++i) {
        P[i].x = __dadd_rn(__dadd_rn(__dmul_rn(c, dx[i]), __dmul_rn(s, dz[i])), r[t1]);
        P[i].y = __dadd_rn(__dadd_rn(__dmul_rn(-s, dx[i]), __dmul_rn(c, dz[i])), r[t3]);
    }
}

// imageBoxOverlap (:229-263), a = detection, b = ground truth
__device__ double ke_image_overlap(const double *d, const double *g, bool crit0) {
    const double x1 = fmax(d[D_X1], g[G_X1]), y1 = fmax(d[D_Y1], g[G_Y1]);
    const double x2 = fmin(d[D_X2], g[G_X2]), y2 = fmin(d[D_Y2], g[G_Y2]);
    const double w = x2 - x1, h = y2 - y1;
    if (w <= 0 || h <= 0) return 0;
    const double inter = __dmul_rn(w, h);
    const double a_area = __dmul_rn(d[D_X2] - d[D_X1], d[D_Y2] - d[D_Y1]);
    const double b_area = __dmul_rn(g[G_X2] - g[G_X1], g[G_Y2] - g[G_Y1]);
    return crit0 ? inter / a_area : inter / __dadd_rn(__dadd_rn(a_area, b_area), -inter);
}

// groundBoxOverlap (:296-316) and box3DOverlap (:319-346).  The union polygon of two overlapping convex polygons
// has the area a + b - inter; disjoint polygons have inter = 0 and the overlap is 0 either way.
__device__ void ke_rotated_overlap(const double *d, const double *g, bool crit0, double *bev, double *o3d) {
    Pt2d gp[4], dp[4];
    ke_polygon(g, G_RY, G_L, G_W, G_T1, G_T3, gp);
    ke_polygon(d, D_RY, D_L, D_W, D_T1, D_T3, dp);
    int n;
    double inter = clip_quads_area(gp, dp, &n);
    inter = n >= 3 ? fabs(inter) : 0.0;
    const double g_area = -shoelace_ccw(gp, 4), d_area = -shoelace_ccw(dp, 4);   // clockwise positive (Boost)
    *bev = crit0 ? inter / d_area : inter / __dadd_rn(__dadd_rn(g_area, d_area), -inter);
    const double ymax = fmin(d[D_T2], g[G_T2]);
    const double ymin = fmax(d[D_T2] - d[D_H], g[G_T2] - g[G_H]);
    const double inter_vol = __dmul_rn(inter, fmax(0.0, ymax - ymin));
    const double det_vol = __dmul_rn(__dmul_rn(d[D_H], d[D_L]), d[D_W]);
    const double gt_vol = __dmul_rn(__dmul_rn(g[G_H], g[G_L]), g[G_W]);
    *o3d = crit0 ? inter_vol / det_vol : inter_vol / __dadd_rn(__dadd_rn(det_vol, gt_vol), -inter_vol);
}

__global__ void ke_flags_kernel(int num_det, const double *__restrict__ det, int *__restrict__ flags) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < num_det; j += gridDim.x * blockDim.x) {
        const double *r = det + (size_t)j * FCN_KITTI_DET_COLS;
        if (r[D_ALPHA] == -10) atomicOr(flags + F_NO_AOS, 1);
        const int c = (int)r[D_CODE];
        if (c < 0 || c > 2) continue;
        if (r[D_X1] >= 0) atomicOr(flags + F_IMAGE + c, 1);
        if (r[D_T1] != -1000) atomicOr(flags + F_GROUND + c, 1);
        if (r[D_T2] != -1000) atomicOr(flags + F_3D + c, 1);
    }
}

__global__ void ke_counts_kernel(int num_images, const int32_t *__restrict__ gt_off, const int32_t *__restrict__ det_off,
                                 long long *__restrict__ pair_cnt, int32_t *__restrict__ word_cnt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > num_images) return;
    if (i == num_images) {                         // the scans' last element is the total
        pair_cnt[i] = 0;
        word_cnt[i] = 0;
        return;
    }
    const long long nd = det_off[i + 1] - det_off[i], ng = gt_off[i + 1] - gt_off[i];
    pair_cnt[i] = nd * ng;
    word_cnt[i] = (int32_t)((nd + 31) / 32);
}

// one thread per pair; ov[m * num_pairs + p] for metric m, pair p = pair_off[i] + j * ng_i + k
__global__ void ke_pairs_kernel(int num_images, long long num_pairs, const double *__restrict__ gt,
                                const double *__restrict__ det, const int32_t *__restrict__ gt_off,
                                const int32_t *__restrict__ det_off, const long long *__restrict__ pair_off,
                                double *__restrict__ ov) {
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < num_pairs;
         p += (long long)gridDim.x * blockDim.x) {
        int lo = 0, hi = num_images - 1;           // the image: last i with pair_off[i] <= p (non-empty images)
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (pair_off[mid] <= p) lo = mid; else hi = mid - 1;
        }
        const int i = lo;
        const long long q = p - pair_off[i];
        const int ng = gt_off[i + 1] - gt_off[i];
        const int j = (int)(q / ng), k = (int)(q % ng);
        const double *d = det + (size_t)(det_off[i] + j) * FCN_KITTI_DET_COLS;
        const double *g = gt + (size_t)(gt_off[i] + k) * FCN_KITTI_GT_COLS;
        const bool crit0 = (int)g[G_CODE] == FCN_KITTI_DONTCARE;
        double bev, o3d;
        ke_rotated_overlap(d, g, crit0, &bev, &o3d);
        ov[p] = ke_image_overlap(d, g, crit0);
        ov[num_pairs + p] = bev;
        ov[2 * num_pairs + p] = o3d;
    }
}

// ------------------------------------------------------------------------------------------------ cleanData
// ignored_gt: 0 counted, 1 neighbour class or beyond the difficulty (matched but not counted), -1 other class
__device__ __forceinline__ int ke_ignored_gt(const double *g, int cls, int diff) {
    const int code = (int)g[G_CODE];
    int valid;
    if (code == cls) valid = 1;
    else if ((cls == FCN_KITTI_PEDESTRIAN && code == FCN_KITTI_PERSON_SITTING) ||
             (cls == FCN_KITTI_CAR && code == FCN_KITTI_VAN)) valid = 0;
    else valid = -1;
    const double height = g[G_Y2] - g[G_Y1];
    const bool ignore = (int)g[G_OCCL] > c_max_occlusion[diff] || g[G_TRUNC] > c_max_truncation[diff] ||
                        height < c_min_height[diff];
    if (valid == 1 && !ignore) return 0;
    if (valid == 0 || (ignore && valid == 1)) return 1;
    return -1;
}

// ignored_det: 1 below the minimum height (any class), 0 the evaluated class, -1 other.  The height is truncated
// to int32 (:446).
__device__ __forceinline__ int ke_ignored_det(const double *d, int cls, int diff) {
    const int height = (int)fabs(d[D_Y1] - d[D_Y2]);
    if (height < c_min_height[diff]) return 1;
    return (int)d[D_CODE] == cls ? 0 : -1;
}

struct KeStat {
    int tp, fp, fn, n_gt;
    double similarity;
};

// computeStatistics (:458-616) for one image.  compute_fp = false (pass 1): TP scores go to `scores` (at most ng of
// them), the rest of the image's ng slots get -inf.  compute_fp = true (pass 2): TP / FP / FN and the AOS sum.
template <bool COMPUTE_FP>
__device__ KeStat ke_image_stats(int m, int cls, int diff, const double *__restrict__ gt, int ng,
                                 const double *__restrict__ det, int nd, const double *__restrict__ ov, int ov_stride,
                                 unsigned *__restrict__ assigned, bool compute_aos, double thresh,
                                 double *__restrict__ scores) {
    KeStat st = {0, 0, 0, 0, 0.0};
    const double min_overlap = c_min_overlap[m][cls];
    for (int w = 0; w < (nd + 31) / 32; ++w) assigned[w] = 0u;
    auto is_assigned = [&](int j) { return (assigned[j >> 5] >> (j & 31)) & 1u; };
    auto assign = [&](int j) { assigned[j >> 5] |= 1u << (j & 31); };
    auto ignored_thresh = [&](int j) { return COMPUTE_FP && det[(size_t)j * FCN_KITTI_DET_COLS + D_SCORE] < thresh; };
    double sim = 0.0;
    int ntp_scores = 0;
    for (int k = 0; k < ng; ++k) {
        const double *g = gt + (size_t)k * FCN_KITTI_GT_COLS;
        const int ig = ke_ignored_gt(g, cls, diff);
        if (ig == 0) ++st.n_gt;
        if (ig == -1) continue;
        int det_idx = -1;
        double valid_detection = KE_NO_DETECTION, max_overlap = 0;
        bool assigned_ignored_det = false;
        for (int j = 0; j < nd; ++j) {
            const double *d = det + (size_t)j * FCN_KITTI_DET_COLS;
            const int idet = ke_ignored_det(d, cls, diff);
            if (idet == -1 || is_assigned(j) || ignored_thresh(j)) continue;
            const double overlap = ov[(size_t)j * ov_stride + k];
            if (!COMPUTE_FP) {
                if (overlap > min_overlap && d[D_SCORE] > valid_detection) {
                    det_idx = j;
                    valid_detection = d[D_SCORE];
                }
            } else if (overlap > min_overlap && (overlap > max_overlap || assigned_ignored_det) && idet == 0) {
                max_overlap = overlap;
                det_idx = j;
                valid_detection = 1;
                assigned_ignored_det = false;
            } else if (overlap > min_overlap && valid_detection == KE_NO_DETECTION && idet == 1) {
                det_idx = j;
                valid_detection = 1;
                assigned_ignored_det = true;
            }
        }
        if (valid_detection == KE_NO_DETECTION && ig == 0) {
            ++st.fn;
        } else if (valid_detection != KE_NO_DETECTION &&
                   (ig == 1 || ke_ignored_det(det + (size_t)det_idx * FCN_KITTI_DET_COLS, cls, diff) == 1)) {
            assign(det_idx);
        } else if (valid_detection != KE_NO_DETECTION) {
            ++st.tp;
            const double *d = det + (size_t)det_idx * FCN_KITTI_DET_COLS;
            if (!COMPUTE_FP) scores[ntp_scores++] = d[D_SCORE];
            if (COMPUTE_FP && compute_aos) sim += (1.0 + cos(g[G_ALPHA] - d[D_ALPHA])) / 2.0;
            assign(det_idx);
        }
    }
    if constexpr (!COMPUTE_FP) {
        for (int k = ntp_scores; k < ng; ++k) scores[k] = -INFINITY;
    } else {
        for (int j = 0; j < nd; ++j) {
            const int idet = ke_ignored_det(det + (size_t)j * FCN_KITTI_DET_COLS, cls, diff);
            if (!(is_assigned(j) || idet == -1 || idet == 1 || ignored_thresh(j))) ++st.fp;
        }
        int nstuff = 0;
        for (int k = 0; k < ng; ++k) {
            if ((int)gt[(size_t)k * FCN_KITTI_GT_COLS + G_CODE] != FCN_KITTI_DONTCARE) continue;
            for (int j = 0; j < nd; ++j) {
                if (is_assigned(j)) continue;
                const int idet = ke_ignored_det(det + (size_t)j * FCN_KITTI_DET_COLS, cls, diff);
                if (idet == -1 || idet == 1 || ignored_thresh(j)) continue;
                if (ov[(size_t)j * ov_stride + k] > min_overlap) {
                    assign(j);
                    ++nstuff;
                }
            }
        }
        st.fp -= nstuff;
        if (compute_aos) st.similarity = (st.tp > 0 || st.fp > 0) ? sim : -1.0;
    }
    return st;
}

// ------------------------------------------------------------------------------------------------ pass 1
__global__ void __launch_bounds__(KE_THREADS)
ke_pass1_kernel(int num_images, int num_gt, long long num_pairs, long long mask_words, const double *__restrict__ gt,
                const double *__restrict__ det, const int32_t *__restrict__ gt_off,
                const int32_t *__restrict__ det_off, const long long *__restrict__ pair_off,
                const int32_t *__restrict__ word_off, const double *__restrict__ ov, unsigned *__restrict__ mask,
                double *__restrict__ scores, int32_t *__restrict__ tp_cnt, int32_t *__restrict__ ngt_cnt,
                int32_t *__restrict__ seg_off) {
    const int e = blockIdx.y, i = blockIdx.x * KE_THREADS + threadIdx.x;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        seg_off[e] = e * num_gt;
        if (e == KE_EVALS - 1) seg_off[KE_EVALS] = KE_EVALS * num_gt;
    }
    if (i >= num_images) return;
    const int m = e / 9, cls = (e / 3) % 3, diff = e % 3;
    const int g0 = gt_off[i], ng = gt_off[i + 1] - g0, d0 = det_off[i], nd = det_off[i + 1] - d0;
    const KeStat st = ke_image_stats<false>(m, cls, diff, gt + (size_t)g0 * FCN_KITTI_GT_COLS, ng,
                                            det + (size_t)d0 * FCN_KITTI_DET_COLS, nd,
                                            ov + m * num_pairs + pair_off[i], ng,
                                            mask + e * mask_words + word_off[i], false, 0.0,
                                            scores + (size_t)e * num_gt + g0);
    tp_cnt[(size_t)e * num_images + i] = st.tp;
    ngt_cnt[(size_t)e * num_images + i] = st.n_gt;
}

// getThresholds (:348-381) on the sorted scores, one thread per evaluation
__global__ void ke_thresholds_kernel(int num_images, int num_gt, const double *__restrict__ sorted,
                                     const int32_t *__restrict__ tp_cnt, const int32_t *__restrict__ ngt_cnt,
                                     double *__restrict__ thresholds, int32_t *__restrict__ n_thr,
                                     int32_t *__restrict__ n_gt_out) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= KE_EVALS) return;
    long long nv = 0, n_gt = 0;
    for (int i = 0; i < num_images; ++i) {
        nv += tp_cnt[(size_t)e * num_images + i];
        n_gt += ngt_cnt[(size_t)e * num_images + i];
    }
    const double *v = sorted + (size_t)e * num_gt;
    const double n_groundtruth = (double)n_gt;
    double current_recall = 0;
    int nt = 0;
    for (long long i = 0; i < nv; ++i) {
        const double l_recall = (double)(i + 1) / n_groundtruth;
        const double r_recall = i < nv - 1 ? (double)(i + 2) / n_groundtruth : l_recall;
        if ((r_recall - current_recall) < (current_recall - l_recall) && i < nv - 1) continue;
        // The reference pushes every selected score into a vector and then indexes a 41-entry one with it; the
        // recall steps bound the selections by 41 (each is at least the previous recall plus 1/40), kept as a guard.
        if (nt < KE_PTS) thresholds[e * KE_PTS + nt] = v[i];
        ++nt;
        current_recall += 1.0 / (KE_PTS - 1.0);
    }
    n_thr[e] = nt < KE_PTS ? nt : KE_PTS;
    n_gt_out[e] = (int32_t)n_gt;
}

// ------------------------------------------------------------------------------------------------ pass 2
__global__ void __launch_bounds__(KE_THREADS)
ke_pass2_kernel(int num_images, long long num_pairs, long long mask_words, const double *__restrict__ gt,
                const double *__restrict__ det, const int32_t *__restrict__ gt_off,
                const int32_t *__restrict__ det_off, const long long *__restrict__ pair_off,
                const int32_t *__restrict__ word_off, const double *__restrict__ ov, const int *__restrict__ flags,
                const double *__restrict__ thresholds, const int32_t *__restrict__ n_thr, unsigned *__restrict__ mask,
                int4 *__restrict__ part_cnt, double *__restrict__ part_sim) {
    __shared__ int s_cnt[3][KE_THREADS];
    __shared__ double s_sim[KE_THREADS];
    const int e = blockIdx.z, t = blockIdx.y, tid = threadIdx.x, i = blockIdx.x * KE_THREADS + tid;
    const int m = e / 9, cls = (e / 3) % 3, diff = e % 3;
    if (t >= n_thr[e]) return;                                    // uniform over the CTA
    const bool compute_aos = m == 0 && flags[F_NO_AOS] == 0;
    KeStat st = {0, 0, 0, 0, -1.0};
    if (i < num_images) {
        const int g0 = gt_off[i], ng = gt_off[i + 1] - g0, d0 = det_off[i], nd = det_off[i + 1] - d0;
        st = ke_image_stats<true>(m, cls, diff, gt + (size_t)g0 * FCN_KITTI_GT_COLS, ng,
                                  det + (size_t)d0 * FCN_KITTI_DET_COLS, nd, ov + m * num_pairs + pair_off[i], ng,
                                  mask + ((long long)e * KE_PTS + t) * mask_words + word_off[i], compute_aos,
                                  thresholds[e * KE_PTS + t], nullptr);
    }
    s_cnt[0][tid] = st.tp;
    s_cnt[1][tid] = st.fp;
    s_cnt[2][tid] = st.fn;
    s_sim[tid] = st.similarity != -1 ? st.similarity : 0.0;      // eval_class skips -1 (:675-676)
    __syncthreads();
    for (int s = KE_THREADS / 2; s > 0; s >>= 1) {
        if (tid < s) {
            for (int c = 0; c < 3; ++c) s_cnt[c][tid] += s_cnt[c][tid + s];
            s_sim[tid] += s_sim[tid + s];
        }
        __syncthreads();
    }
    if (tid == 0) {
        const size_t slot = ((size_t)e * KE_PTS + t) * gridDim.x + blockIdx.x;
        part_cnt[slot] = make_int4(s_cnt[0][0], s_cnt[1][0], s_cnt[2][0], 0);
        part_sim[slot] = s_sim[0];
    }
}

// std::max_element: the first element that no later element exceeds
__device__ double ke_suffix_max(const double *v, int from) {
    int best = from;
    for (int i = from + 1; i < KE_PTS; ++i)
        if (v[best] < v[i]) best = i;
    return v[best];
}

// eval_class tail (:680-699) and the AP line of saveAndPlotPlots (:716-720), one thread per evaluation
__global__ void ke_finalize_kernel(int nblk, const int *__restrict__ flags, const int32_t *__restrict__ n_thr,
                                   const int32_t *__restrict__ n_gt, const int4 *__restrict__ part_cnt,
                                   const double *__restrict__ part_sim, fcn_kitti_eval_result *__restrict__ out) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= KE_EVALS) return;
    const int m = e / 9, cls = (e / 3) % 3, diff = e % 3;
    const bool compute_aos = m == 0 && flags[F_NO_AOS] == 0;
    double *prec = out->precision[m][cls][diff];
    double *aos = out->aos[cls][diff];
    for (int i = 0; i < KE_PTS; ++i) prec[i] = 0.0;
    if (m == 0)
        for (int i = 0; i < KE_PTS; ++i) aos[i] = 0.0;
    const int nt = n_thr[e];
    for (int t = 0; t < nt; ++t) {
        long long tp = 0, fp = 0;
        double sim = 0.0;
        for (int b = 0; b < nblk; ++b) {
            const size_t slot = ((size_t)e * KE_PTS + t) * nblk + b;
            tp += part_cnt[slot].x;
            fp += part_cnt[slot].y;
            sim += part_sim[slot];
        }
        prec[t] = (double)tp / (double)(tp + fp);
        if (compute_aos) aos[t] = sim / (double)(tp + fp);
    }
    for (int t = 0; t < nt; ++t) {
        prec[t] = ke_suffix_max(prec, t);
        if (compute_aos) aos[t] = ke_suffix_max(aos, t);
    }
    float sum = 0.f, sum_aos = 0.f;
    for (int i = 0; i < KE_PTS; i += 4) {
        sum = (float)((double)sum + prec[i]);                     // float += double (:716-719)
        if (m == 0) sum_aos = (float)((double)sum_aos + aos[i]);
    }
    out->ap[m][cls][diff] = sum / 11 * 100;
    if (m == 0) out->ap_aos[cls][diff] = sum_aos / 11 * 100;
    out->n_thresholds[m][cls][diff] = nt;
    out->n_gt[m][cls][diff] = n_gt[e];
    if (diff == 0) out->evaluated[m][cls] = flags[3 * m + cls];
    if (e == 0) {
        out->compute_aos = flags[F_NO_AOS] == 0;
        out->reserved = 0;
    }
}

// ------------------------------------------------------------------------------------------------ host side
struct KeWs {
    int *flags;
    long long *pair_cnt, *pair_off;
    int32_t *word_cnt, *word_off, *tp_cnt, *ngt_cnt, *seg_off, *n_thr, *n_gt;
    double *ov, *scores, *sorted, *thresholds, *part_sim;
    int4 *part_cnt;
    unsigned *mask;
    void *temp;
    size_t temp_bytes;
};

struct KeSizes {
    long long num_pairs, mask_words;
};

static int ke_nblk(int num_images) { return std::max(1, ceil_div(num_images, KE_THREADS)); }

static cudaError_t ke_layout(const fcn_kitti_eval_args *a, const KeSizes &sz, Carve &c, KeWs &w) {
    const size_t N = (size_t)a->num_images, G = (size_t)a->num_gt;
    size_t t_sort = 0, t_scan32 = 0, t_scan64 = 0;
    const int items = (int)(KE_EVALS * G);
    cudaError_t e = cub::DeviceSegmentedRadixSort::SortKeysDescending(
        nullptr, t_sort, (const double *)nullptr, (double *)nullptr, std::max(items, 1), KE_EVALS, (const int32_t *)nullptr,
        (const int32_t *)nullptr);
    if (e != cudaSuccess) return e;
    e = cub::DeviceScan::ExclusiveSum(nullptr, t_scan32, (int32_t *)nullptr, (int32_t *)nullptr, (int)N + 1);
    if (e != cudaSuccess) return e;
    e = cub::DeviceScan::ExclusiveSum(nullptr, t_scan64, (long long *)nullptr, (long long *)nullptr, (int)N + 1);
    if (e != cudaSuccess) return e;
    w.temp_bytes = std::max(t_sort, std::max(t_scan32, t_scan64));
    const size_t parts = (size_t)KE_EVALS * KE_PTS * ke_nblk(a->num_images);
    w.flags = (int *)c.take(F_COUNT * 4);
    w.pair_cnt = (long long *)c.take((N + 1) * 8);
    w.pair_off = (long long *)c.take((N + 1) * 8);
    w.word_cnt = (int32_t *)c.take((N + 1) * 4);
    w.word_off = (int32_t *)c.take((N + 1) * 4);
    w.ov = (double *)c.take(3 * (size_t)sz.num_pairs * 8);
    w.tp_cnt = (int32_t *)c.take(KE_EVALS * N * 4);
    w.ngt_cnt = (int32_t *)c.take(KE_EVALS * N * 4);
    w.seg_off = (int32_t *)c.take((KE_EVALS + 1) * 4);
    w.scores = (double *)c.take(KE_EVALS * G * 8);
    w.sorted = (double *)c.take(KE_EVALS * G * 8);
    w.thresholds = (double *)c.take(KE_EVALS * KE_PTS * 8);
    w.n_thr = (int32_t *)c.take(KE_EVALS * 4);
    w.n_gt = (int32_t *)c.take(KE_EVALS * 4);
    w.mask = (unsigned *)c.take((size_t)KE_EVALS * KE_PTS * (size_t)sz.mask_words * 4);
    w.part_cnt = (int4 *)c.take(parts * sizeof(int4));
    w.part_sim = (double *)c.take(parts * 8);
    w.temp = c.take(w.temp_bytes);
    return cudaSuccess;
}

// Host-side checks shared by every entry: counts, pointers and the host copies of the offsets.  Fills the pair and
// mask-word totals.
static int ke_check(const fcn_kitti_eval_args *a, const char *fn, KeSizes &sz) {
    if (a == nullptr) return invalid(fn, "NULL args");
    if (a->num_images < 0 || a->num_gt < 0 || a->num_det < 0)
        return invalid(fn, "negative count (num_images, num_gt, num_det must be >= 0)");
    if (a->num_gt > (1 << 26) || a->num_det > (1 << 28) || a->num_images > (1 << 26))
        return invalid(fn, "too many records (num_gt <= 2^26, num_det <= 2^28, num_images <= 2^26)");
    if (!a->host_gt_offsets || !a->host_det_offsets) return invalid(fn, "NULL host offsets");
    if (!a->gt_offsets || !a->det_offsets || (a->num_gt > 0 && !a->gt) || (a->num_det > 0 && !a->det))
        return invalid(fn, "NULL pointer");
    const int32_t *go = a->host_gt_offsets, *dof = a->host_det_offsets;
    if (!offsets_ok(go, a->num_images, a->num_gt) || !offsets_ok(dof, a->num_images, a->num_det))
        return invalid(fn, "offsets must start at 0, must not decrease and must end at num_gt and num_det");
    long long pairs = 0, words = 0;
    for (int i = 0; i < a->num_images; ++i) {
        const long long ng = (long long)go[i + 1] - go[i], nd = (long long)dof[i + 1] - dof[i];
        pairs += ng * nd;
        words += (nd + 31) / 32;
    }
    sz.num_pairs = pairs;
    sz.mask_words = words;
    return FCN_OK;
}

static int ke_prepare(const fcn_kitti_eval_args *a, const char *fn, KeWs &w, KeSizes &sz) {
    const int st = ke_check(a, fn, sz);
    if (st != FCN_OK) return st;
    if (!a->workspace || !a->result) return invalid(fn, "NULL workspace or result");
    return carve_workspace(fn, "kitti_eval", a->workspace, a->workspace_bytes,
                           [&](Carve &c) { return ke_layout(a, sz, c, w); });
}

}  // namespace fcn

using namespace fcn;

extern "C" long long fcn_kitti_eval_workspace_bytes(const fcn_kitti_eval_args *a) {
    KeSizes sz;
    if (ke_check(a, __func__, sz) != FCN_OK) return -1;
    KeWs w;
    return workspace_size(__func__, [&](Carve &c) { return ke_layout(a, sz, c, w); });
}

extern "C" int fcn_kitti_eval_overlaps(const fcn_kitti_eval_args *a, fcn_stream_t stream) {
    KeWs w;
    KeSizes sz;
    const int st = ke_prepare(a, __func__, w, sz);
    if (st != FCN_OK) return st;
    cudaStream_t s = (cudaStream_t)stream;
    const int N = a->num_images;
    FCN_CUDA(cudaMemsetAsync(w.flags, 0, F_COUNT * 4, s));
    if (a->num_det > 0) {
        ke_flags_kernel<<<std::min(ceil_div(a->num_det, 256), sm_count() * 4), 256, 0, s>>>(a->num_det, a->det, w.flags);
        FCN_LAUNCH_CHECK();
    }
    ke_counts_kernel<<<ceil_div(N + 1, 256), 256, 0, s>>>(N, a->gt_offsets, a->det_offsets, w.pair_cnt, w.word_cnt);
    FCN_LAUNCH_CHECK();
    FCN_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, w.temp_bytes, w.pair_cnt, w.pair_off, N + 1, s));
    FCN_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, w.temp_bytes, w.word_cnt, w.word_off, N + 1, s));
    if (sz.num_pairs > 0) {
        const int grid = (int)std::min<long long>((sz.num_pairs + 255) / 256, (long long)sm_count() * 16);
        ke_pairs_kernel<<<grid, 256, 0, s>>>(N, sz.num_pairs, a->gt, a->det, a->gt_offsets, a->det_offsets,
                                             w.pair_off, w.ov);
        FCN_LAUNCH_CHECK();
    }
    return FCN_OK;
}

extern "C" int fcn_kitti_eval_thresholds(const fcn_kitti_eval_args *a, fcn_stream_t stream) {
    KeWs w;
    KeSizes sz;
    const int st = ke_prepare(a, __func__, w, sz);
    if (st != FCN_OK) return st;
    cudaStream_t s = (cudaStream_t)stream;
    const int N = a->num_images, G = a->num_gt;
    if (N > 0) {
        ke_pass1_kernel<<<dim3(ke_nblk(N), KE_EVALS), KE_THREADS, 0, s>>>(
            N, G, sz.num_pairs, sz.mask_words, a->gt, a->det, a->gt_offsets, a->det_offsets, w.pair_off, w.word_off,
            w.ov, w.mask, w.scores, w.tp_cnt, w.ngt_cnt, w.seg_off);
        FCN_LAUNCH_CHECK();
    }
    if (G > 0) {
        FCN_CUDA(cub::DeviceSegmentedRadixSort::SortKeysDescending(w.temp, w.temp_bytes, w.scores, w.sorted,
                                                                   KE_EVALS * G, KE_EVALS, w.seg_off, w.seg_off + 1,
                                                                   0, 64, s));
    }
    ke_thresholds_kernel<<<1, 32, 0, s>>>(N, G, w.sorted, w.tp_cnt, w.ngt_cnt, w.thresholds, w.n_thr, w.n_gt);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

extern "C" int fcn_kitti_eval_statistics(const fcn_kitti_eval_args *a, fcn_stream_t stream) {
    KeWs w;
    KeSizes sz;
    const int st = ke_prepare(a, __func__, w, sz);
    if (st != FCN_OK) return st;
    cudaStream_t s = (cudaStream_t)stream;
    const int N = a->num_images, nblk = ke_nblk(N);
    if (N > 0) {
        ke_pass2_kernel<<<dim3(nblk, KE_PTS, KE_EVALS), KE_THREADS, 0, s>>>(
            N, sz.num_pairs, sz.mask_words, a->gt, a->det, a->gt_offsets, a->det_offsets, w.pair_off, w.word_off,
            w.ov, w.flags, w.thresholds, w.n_thr, w.mask, w.part_cnt, w.part_sim);
        FCN_LAUNCH_CHECK();
    }
    ke_finalize_kernel<<<1, 32, 0, s>>>(N > 0 ? nblk : 0, w.flags, w.n_thr, w.n_gt, w.part_cnt, w.part_sim,
                                         a->result);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}
