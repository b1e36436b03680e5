// Per-row forward terms of the detection losses and metrics (det_base.py:414-525), shared by the training loss
// kernels (loss.cu: forward + hand-derived gradient, float atomics) and the validation kernels (validate.cu: forward
// only, fixed-slot reductions).  Every helper is force-inlined, so both callers compile the same instruction
// sequence for a term; loss.cu's kernels come out with the SASS they had before these terms were moved here.
#pragma once
#include "box_iou.cuh"
#include "common.cuh"

namespace fcn {

constexpr int LOSS_MAX_BINS = 32;
constexpr float LOSS_PI = 3.14159265358979323846f;

// accumulator slots of one row: the seven loss terms, the three accuracies, the three IoU metrics
enum { A_CLS = 0, A_CENTER, A_HCLS, A_HRES, A_SCLS, A_SRES, A_CORNER, A_CLSACC, A_HACC, A_SACC, A_IOU2, A_IOU3, A_IOUGT, A_N };

__device__ __forceinline__ float huber(float a_abs, float delta) {
    const float q = fminf(a_abs, delta);
    return 0.5f * q * q + delta * (a_abs - q);
}

// corners of models/model_util.py:48-72 (x: +-l/2, y: +-h/2, z: +-w/2; rotation about y)
__device__ __forceinline__ void corners_of(const float *ctr, float heading, const float *size, float *c) {
    const float l = size[0], w = size[1], h = size[2];
    const float cs = cosf(heading), sn = sinf(heading);
    const float sx[8] = {1, 1, -1, -1, 1, 1, -1, -1}, sy[8] = {1, 1, 1, 1, -1, -1, -1, -1}, sz[8] = {1, -1, -1, 1, 1, -1, -1, 1};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float x = sx[j] * l * 0.5f, y = sy[j] * h * 0.5f, z = sz[j] * w * 0.5f;
        c[3 * j + 0] = cs * x + sn * z + ctr[0];
        c[3 * j + 1] = y + ctr[1];
        c[3 * j + 2] = -sn * x + cs * z + ctr[2];
    }
}

// two-class softmax of the classification logits (det_base.py:383)
__device__ __forceinline__ void softmax2(const float *cl, float &p0, float &p1) {
    const float m = fmaxf(cl[0], cl[1]);
    const float e0 = expf(cl[0] - m), e1 = expf(cl[1] - m);
    p0 = e0 / (e0 + e1);
    p1 = e1 / (e0 + e1);
}

// focal term -alpha (1 - pt)^2 log(pt + 1e-14) of one row with label != -1 (common.py:217-232); lg = log(pt + 1e-14)
__device__ __forceinline__ float focal_term(float pt, float alpha, float &lg) {
    lg = logf(pt + 1e-14f);
    return -alpha * (1.f - pt) * (1.f - pt) * lg;
}

// width of one heading bin: 2 pi / NH rounded once from double, as the model's python constant enters its float32
// tensor arithmetic (and as decode.cuh computes it).  float32(2 pi) / NH differs by 1 ulp for NH = 9, 11, 13, ...
__device__ __forceinline__ float heading_bin_width(int NH) {
    return (float)(2.0 * 3.14159265358979323846 / (double)NH);
}

// angle_encode (box_transform.py:34-47): heading class and normalised residual of a GT heading
__device__ __forceinline__ int angle_encode(float hgt, int NH, float &hres_lab) {
    const float two_pi = 2.f * LOSS_PI, apc = heading_bin_width(NH);
    float g = fmodf(hgt, two_pi);
    if (g < 0.f) g += two_pi;                                  // python-style modulo
    float shifted = fmodf(g + apc * 0.5f, two_pi);
    if (shifted < 0.f) shifted += two_pi;
    const int hc = min(max((int)floorf(shifted / apc), 0), NH - 1);
    hres_lab = (shifted - ((float)hc * apc + apc * 0.5f)) / (apc * 0.5f);
    return hc;
}

// angle_decode (box_transform.py:50-58) of class c with normalised residual r
__device__ __forceinline__ float angle_decode(int c, float r, float apc) {
    float ang = (float)c * apc + r * (apc * 0.5f);
    if (ang > LOSS_PI) ang -= 2.f * LOSS_PI;
    return ang;
}

// log-sum-exp pieces of a softmax row: returns sum_i exp(s_i - mx), mx = max_i s_i
__device__ __forceinline__ float softmax_denom(const float *s, int n, float &mx) {
    mx = s[0];
    for (int i = 1; i < n; ++i) mx = fmaxf(mx, s[i]);
    float sum = 0.f;
    for (int i = 0; i < n; ++i) sum += expf(s[i] - mx);
    return sum;
}

// The 14 values of a batch (det_base.py:505-523) from its summed row terms acc[A_*] and its foreground and
// non-ignored row counts; `a` is the caller's settings record (fcn_loss_args or fcn_val_batch_args).
//   out[0..7]  = total, cls, center, head_cls, head_res, size_cls, size_res, corners
//   out[8..13] = cls_acc, head_acc, size_acc, IoU_2D, IoU_3D, IoU_>=thresh   (NaN IoU values when with_iou == 0)
// Every product, sum and quotient is rounded on its own, as the reference's float32 tensor operations round them:
// the total in Python's evaluation order of det_base.py:468-474, and each accuracy as get_accuracy
// (utils/utils.py:28-48) forms it, correct.sum() * float32(1.0 / n).  The explicit _rn intrinsics keep nvcc from
// contracting the total into FFMAs.
template <class Args>
__device__ __forceinline__ void loss_final_values(const Args &a, const float *acc, float nfg_raw, float nkeep_raw,
                                                  float *out) {
    const float nfg = fmaxf(nfg_raw, 1.f), nkeep = fmaxf(nkeep_raw, 1.f);
    const float cls = __fdiv_rn(acc[A_CLS], __fadd_rn(nfg_raw, 1e-14f));   // loss.sum() / (num_fg + 1e-14)
    const float center = __fdiv_rn(acc[A_CENTER], nfg), hcls = __fdiv_rn(acc[A_HCLS], nfg);
    const float hres = __fdiv_rn(acc[A_HRES], nfg), scls = __fdiv_rn(acc[A_SCLS], nfg);
    const float sres = __fdiv_rn(acc[A_SRES], nfg), corner = __fdiv_rn(acc[A_CORNER], nfg);
    float box = __fadd_rn(__fadd_rn(center, hcls), scls);
    box = __fadd_rn(box, __fmul_rn(a.w_head_reg, hres));
    box = __fadd_rn(box, __fmul_rn(a.w_size_reg, sres));
    box = __fadd_rn(box, __fmul_rn(a.w_corner, corner));
    out[0] = __fadd_rn(cls, __fmul_rn(a.w_box, box));
    out[1] = cls; out[2] = center; out[3] = hcls; out[4] = hres; out[5] = scls; out[6] = sres; out[7] = corner;
    out[8] = __fmul_rn(acc[A_CLSACC], __double2float_rn(1.0 / (double)nkeep));
    out[9] = __fmul_rn(acc[A_HACC], __double2float_rn(1.0 / (double)nfg));
    out[10] = __fmul_rn(acc[A_SACC], __double2float_rn(1.0 / (double)nfg));
    const float nan = __int_as_float(0x7fc00000);
    out[11] = a.with_iou ? __fdiv_rn(acc[A_IOU2], nfg) : nan;
    out[12] = a.with_iou ? __fdiv_rn(acc[A_IOU3], nfg) : nan;
    out[13] = a.with_iou ? __fdiv_rn(acc[A_IOUGT], nfg) : nan;
}

}  // namespace fcn
