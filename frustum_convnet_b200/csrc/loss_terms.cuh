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

}  // namespace fcn
