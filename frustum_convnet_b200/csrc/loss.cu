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
#include <type_traits>

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

// One thread per row: row r's loss terms and its logit gradients to a.dcls / a.dreg, then the CTA's sums of the
// A_N terms.  ORDERED (fcn_det_loss_deterministic): each warp's sums (a fixed butterfly) are added in warp order and
// the CTA's sums go to its slot dst[CTA][A_N] with plain stores; else they are added to dst[A_N] by atomics.  dcls /
// dreg never read the sums and are the same in both.
template <bool ORDERED>
__global__ void __launch_bounds__(128)
det_loss_rows_kernel(const __grid_constant__ fcn_loss_args a, const float *__restrict__ counts, float *__restrict__ dst) {
    __shared__ std::conditional_t<ORDERED, float[4][A_N], float[A_N]> s_acc;    // per warp, or atomics
    if constexpr (!ORDERED) {
        if (threadIdx.x < A_N) s_acc[threadIdx.x] = 0.f;
        __syncthreads();
    }
    const int N = a.B * a.T2, NH = a.NH, NS = a.NS, W = 3 + 2 * NH + 4 * NS;
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    float v[A_N];
#pragma unroll
    for (int i = 0; i < A_N; ++i) v[i] = 0.f;
    if (r < N) {
        const int b = r / a.T2, t = r - b * a.T2;
        const long long lab = a.cls_label[r];
        const float nfg = fmaxf(counts[0], 1.f), inv_fg = 1.f / nfg;
        const float *cl = a.cls + (size_t)r * 2, *o = a.reg + (size_t)r * W;
        float *dc = a.dcls + (size_t)r * 2, *dr = a.dreg + (size_t)r * W;
        for (int i = 0; i < W; ++i) dr[i] = 0.f;
        // ---------------- focal classification loss (all rows with label != -1), common.py:217-232
        float p0, p1;
        softmax2(cl, p0, p1);
        float d0 = 0.f, d1 = 0.f;
        if (lab != -1) {
            const int tl = lab >= 1 ? 1 : 0;
            const float alpha = tl == 0 ? 0.75f : 0.25f;
            const float pt = tl == 0 ? p0 : p1;
            float lg;
            v[A_CLS] = focal_term(pt, alpha, lg);
            // d/dpt [ -alpha (1-pt)^2 log(pt+eps) ]
            const float dpt = -alpha * (-2.f * (1.f - pt) * lg + (1.f - pt) * (1.f - pt) / (pt + 1e-14f));
            const float scale = dpt / (counts[0] + 1e-14f);           // loss.sum() / (num_fg + 1e-14)
            // dpt/dc_k = pt (delta_kt - p_k)
            d0 = scale * pt * ((tl == 0 ? 1.f : 0.f) - p0);
            d1 = scale * pt * ((tl == 1 ? 1.f : 0.f) - p1);
            v[A_CLSACC] = ((p1 > p0 ? 1 : 0) == (int)lab) ? 1.f : 0.f;   // argmax: first maximum on ties
        }
        dc[0] = d0; dc[1] = d1;
        if (lab == 1) {
            // ---------------- labels of this frustum, box_transform.py:15-25
            const float cgt[3] = {a.box3d_center[b * 3], a.box3d_center[b * 3 + 1], a.box3d_center[b * 3 + 2]};
            const float ref[3] = {a.center_ref2[((size_t)b * 3 + 0) * a.T2 + t], a.center_ref2[((size_t)b * 3 + 1) * a.T2 + t],
                                  a.center_ref2[((size_t)b * 3 + 2) * a.T2 + t]};
            const float hgt = a.box3d_heading[b];
            const float sgt[3] = {a.box3d_size[b * 3], a.box3d_size[b * 3 + 1], a.box3d_size[b * 3 + 2]};
            const int sc = (int)a.size_class[b];
            const float apc = heading_bin_width(NH);
            float hres_lab;
            const int hc = angle_encode(hgt, NH, hres_lab);
            const float *ctr = o, *hs = o + 3, *hr = hs + NH, *ss = hr + NH, *sr = ss + NS;
            float ex[3];
#pragma unroll
            for (int i = 0; i < 3; ++i) ex[i] = a.mean_size[sc * 3 + i];
            const float wb = a.w_box * inv_fg;                         // weight of a box term of ONE fg row in the total
            // ---------------- centre Huber loss (delta 3) on the distance
            {
                float dv[3], d2 = 0.f;
#pragma unroll
                for (int i = 0; i < 3; ++i) { dv[i] = (cgt[i] - ref[i]) - ctr[i]; d2 += dv[i] * dv[i]; }
                const float d = sqrtf(d2);
                v[A_CENTER] = huber(d, 3.f);
                const float gd = d > 0.f ? fminf(d, 3.f) / d : 0.f;   // dh/dd * 1/d
#pragma unroll
                for (int i = 0; i < 3; ++i) dr[i] += wb * gd * (-dv[i]);
            }
            // ---------------- heading class CE + residual Huber (delta 1)
            int h_arg = 0;
            {
                float mx;
                const float sum = softmax_denom(hs, NH, mx);
                v[A_HCLS] = -(hs[hc] - mx - logf(sum));
                float best = -1.f;
                for (int i = 0; i < NH; ++i) {
                    const float p = expf(hs[i] - mx) / sum;
                    dr[3 + i] += wb * (p - (i == hc ? 1.f : 0.f));
                    if (p > best) { best = p; h_arg = i; }
                }
                v[A_HACC] = h_arg == hc ? 1.f : 0.f;
                const float e = hr[hc] - hres_lab;
                v[A_HRES] = huber(fabsf(e), 1.f);
                dr[3 + NH + hc] += wb * a.w_head_reg * fmaxf(-1.f, fminf(1.f, e));
            }
            // ---------------- size class CE + residual Huber (delta 1) on the norm
            int s_arg = 0;
            {
                float mx;
                const float sum = softmax_denom(ss, NS, mx);
                v[A_SCLS] = -(ss[sc] - mx - logf(sum));
                float best = -1.f;
                for (int i = 0; i < NS; ++i) {
                    const float p = expf(ss[i] - mx) / sum;
                    dr[3 + 2 * NH + i] += wb * (p - (i == sc ? 1.f : 0.f));
                    if (p > best) { best = p; s_arg = i; }
                }
                v[A_SACC] = s_arg == sc ? 1.f : 0.f;
                float dv[3], d2 = 0.f;
#pragma unroll
                for (int i = 0; i < 3; ++i) { dv[i] = (sgt[i] - ex[i]) / ex[i] - sr[sc * 3 + i]; d2 += dv[i] * dv[i]; }
                const float d = sqrtf(d2);
                v[A_SRES] = huber(d, 1.f);
                const float gd = d > 0.f ? fminf(d, 1.f) / d : 0.f;
#pragma unroll
                for (int i = 0; i < 3; ++i) dr[3 + 2 * NH + NS + sc * 3 + i] += wb * a.w_size_reg * gd * (-dv[i]);
            }
            // ---------------- corner loss (det_base.py:449-461): predicted box with the GT class labels
            {
                const float cp[3] = {ref[0] + ctr[0], ref[1] + ctr[1], ref[2] + ctr[2]};
                const float ang = angle_decode(hc, hr[hc], apc);
                float sz[3];
#pragma unroll
                for (int i = 0; i < 3; ++i) sz[i] = sr[sc * 3 + i] * ex[i] + ex[i];
                float P[24], G[24], F[24];
                corners_of(cp, ang, sz, P);
                corners_of(cgt, hgt, sgt, G);
                corners_of(cgt, hgt + LOSS_PI, sgt, F);
                float dg = 0.f, df = 0.f, ng[8], nf[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    float a2 = 0.f, b2 = 0.f;
#pragma unroll
                    for (int k = 0; k < 3; ++k) {
                        const float x = P[3 * j + k] - G[3 * j + k], y = P[3 * j + k] - F[3 * j + k];
                        a2 += x * x; b2 += y * y;
                    }
                    ng[j] = sqrtf(a2); nf[j] = sqrtf(b2);
                    dg += ng[j]; df += nf[j];
                }
                dg *= 0.125f; df *= 0.125f;
                const bool use_g = dg <= df;
                const float D = use_g ? dg : df;
                v[A_CORNER] = huber(D, 1.f);
                const float gD = wb * a.w_corner * fminf(D, 1.f) * 0.125f;   // dL/dD * dD/d||.||_j
                const float cs = cosf(ang), sn = sinf(ang);
                const float sx[8] = {1, 1, -1, -1, 1, 1, -1, -1}, sy[8] = {1, 1, 1, 1, -1, -1, -1, -1},
                            szz[8] = {1, -1, -1, 1, 1, -1, -1, 1};
                float gc[3] = {0.f, 0.f, 0.f}, gth = 0.f, gl = 0.f, gw = 0.f, gh = 0.f;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float nrm = use_g ? ng[j] : nf[j];
                    if (!(nrm > 0.f)) continue;
                    const float *Tg = use_g ? G : F;
                    const float gx = gD * (P[3 * j] - Tg[3 * j]) / nrm, gy = gD * (P[3 * j + 1] - Tg[3 * j + 1]) / nrm,
                                gz = gD * (P[3 * j + 2] - Tg[3 * j + 2]) / nrm;
                    gc[0] += gx; gc[1] += gy; gc[2] += gz;
                    const float x = sx[j] * sz[0] * 0.5f, z = szz[j] * sz[1] * 0.5f;
                    gth += gx * (-sn * x + cs * z) + gz * (-cs * x - sn * z);
                    gl += (gx * cs - gz * sn) * sx[j] * 0.5f;
                    gw += (gx * sn + gz * cs) * szz[j] * 0.5f;
                    gh += gy * sy[j] * 0.5f;
                }
#pragma unroll
                for (int i = 0; i < 3; ++i) dr[i] += gc[i];
                dr[3 + NH + hc] += gth * (apc * 0.5f);
                dr[3 + 2 * NH + NS + sc * 3 + 0] += gl * ex[0];
                dr[3 + 2 * NH + NS + sc * 3 + 1] += gw * ex[1];
                dr[3 + 2 * NH + NS + sc * 3 + 2] += gh * ex[2];
                // ---------------- IoU metrics: predicted box with the PREDICTED class labels (det_base.py:488-500)
                if (a.with_iou) {
                    const float angp = angle_decode(h_arg, hr[h_arg], apc);
                    float szp[3];
#pragma unroll
                    for (int i = 0; i < 3; ++i) szp[i] = sr[s_arg * 3 + i] * a.mean_size[s_arg * 3 + i] + a.mean_size[s_arg * 3 + i];
                    corners_of(cp, angp, szp, P);
                    float iou[2];
                    rbbox_iou_pair(P, G, iou);
                    v[A_IOU2] = iou[0];
                    v[A_IOU3] = iou[1];
                    v[A_IOUGT] = iou[1] >= a.iou_thresh ? 1.f : 0.f;
                }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < A_N; ++i) {
        float x = v[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
        if constexpr (ORDERED) {
            if ((threadIdx.x & 31) == 0) s_acc[threadIdx.x / 32][i] = x;
        } else {
            if ((threadIdx.x & 31) == 0 && x != 0.f) atomicAdd(&s_acc[i], x);
        }
    }
    __syncthreads();
    if constexpr (ORDERED) {
        if (threadIdx.x < A_N)
            dst[(size_t)blockIdx.x * A_N + threadIdx.x] =
                ((s_acc[0][threadIdx.x] + s_acc[1][threadIdx.x]) + s_acc[2][threadIdx.x]) + s_acc[3][threadIdx.x];
    } else {
        if (threadIdx.x < A_N && s_acc[threadIdx.x] != 0.f) atomicAdd(&dst[threadIdx.x], s_acc[threadIdx.x]);
    }
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

// the argument checks of both loss entries, reported as errors of the entry `fn`
static int loss_args_check(const char *fn, const fcn_loss_args *args) {
    if (args == nullptr) return invalid(fn, "args is NULL");
    const fcn_loss_args &a = *args;
    if (!(a.B >= 1 && a.T2 >= 1 && a.NH >= 1 && a.NH <= LOSS_MAX_BINS && a.NS >= 1 && a.NS <= LOSS_MAX_BINS))
        return invalid(fn, "bad sizes");
    if (!(a.cls && a.reg && a.center_ref2 && a.cls_label && a.box3d_center && a.box3d_heading && a.box3d_size &&
          a.size_class && a.mean_size && a.dcls && a.dreg && a.out && a.scratch))
        return invalid(fn, "NULL pointer");
    return FCN_OK;
}

extern "C" int fcn_det_loss(const fcn_loss_args *args, fcn_stream_t stream) {
    if (int rc = loss_args_check(__func__, args)) return rc;
    const fcn_loss_args &a = *args;
    cudaStream_t st = (cudaStream_t)stream;
    const int N = a.B * a.T2;
    float *counts = a.scratch, *acc = a.scratch + 2;
    FCN_CUDA(cudaMemsetAsync(a.scratch, 0, sizeof(float) * (2 + A_N), st));
    det_loss_count_kernel<<<min(ceil_div(N, 256), 64), 256, 0, st>>>(N, (const long long *)a.cls_label, counts);
    FCN_LAUNCH_CHECK();
    det_loss_rows_kernel<false><<<ceil_div(N, 128), 128, 0, st>>>(a, counts, acc);
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
    if (int rc = loss_args_check(__func__, args)) return rc;
    const fcn_loss_args &a = *args;
    FCN_REQUIRE(det_loss_rows_ok((long long)a.B * a.T2), "more than 2^24 rows: the float row counts would not be exact");
    cudaStream_t st = (cudaStream_t)stream;
    const int N = a.B * a.T2, nblk = ceil_div(N, 128);
    float *counts = a.scratch, *acc = a.scratch + 2, *slots = a.scratch + 16;
    FCN_CUDA(cudaMemsetAsync(a.scratch, 0, sizeof(float) * 2, st));
    det_loss_count_kernel<<<min(ceil_div(N, 256), 64), 256, 0, st>>>(N, (const long long *)a.cls_label, counts);
    FCN_LAUNCH_CHECK();
    det_loss_rows_kernel<true><<<nblk, 128, 0, st>>>(a, counts, slots);
    FCN_LAUNCH_CHECK();
    det_loss_slots_kernel<<<1, 32, 0, st>>>(nblk, slots, acc);
    FCN_LAUNCH_CHECK();
    det_loss_final_kernel<<<1, 32, 0, st>>>(a, counts, acc, a.out);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}
