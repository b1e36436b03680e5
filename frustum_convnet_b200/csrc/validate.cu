// Validation pass on the device (C ABI section 12): the eval-mode losses and metrics of det_base.py:414-525 read
// straight from the fused forward's pitched head logits, appended to an epoch table without a host sync, and the
// float64 AverageMeter replay of utils/utils.py:51-67 at the end of the epoch.
//   val_rows_kernel   : one thread per (frustum, position) row, the forward terms of loss_terms.cuh; each CTA
//                       writes its 15 sums (13 terms, nfg, nkeep) to its own slot of `partials`
//   val_final_kernel  : one warp sums the slots in CTA order, forms the 14 values as fcn_det_loss does
//                       (loss_final_values) and appends one table row at the index taken from the device counter
//   val_finalize_kernel: one thread per meter replays sum += val * n, count += n (count from 1e-14) in row order
//   train_states_append_kernel: appends a training step's fcn_det_loss result block as one row of the same table
// No float atomics anywhere, so a batch gives the same bits on every run, stream and graph replay.
#include "loss_terms.cuh"

namespace fcn {

constexpr int VAL_THREADS = 128;
constexpr int VAL_SLOT = 16;           // floats per CTA slot: A_N terms, nfg, nkeep, pad
constexpr int VAL_NFG = A_N, VAL_NKEEP = A_N + 1;

__global__ void __launch_bounds__(VAL_THREADS) val_rows_kernel(const __grid_constant__ fcn_val_batch_args a) {
    __shared__ float s_warp[VAL_THREADS / 32][VAL_SLOT];
    const int N = a.B * a.T2, NH = a.NH, NS = a.NS;
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    float v[VAL_SLOT];
#pragma unroll
    for (int i = 0; i < VAL_SLOT; ++i) v[i] = 0.f;
    if (r < N) {
        const int b = r / a.T2, t = r - b * a.T2;
        const long long lab = a.cls_label[r];
        const float *cl = a.logits + ((size_t)b * a.logit_pitch + t) * a.ld_logit, *o = cl + 2;
        if (lab != -1) {
            float p0, p1, lg;
            softmax2(cl, p0, p1);
            const int tl = lab >= 1 ? 1 : 0;
            v[A_CLS] = focal_term(tl == 0 ? p0 : p1, tl == 0 ? 0.75f : 0.25f, lg);
            v[A_CLSACC] = ((p1 > p0 ? 1 : 0) == (int)lab) ? 1.f : 0.f;   // argmax: first maximum on ties
            v[VAL_NKEEP] = 1.f;
        }
        if (lab == 1) {
            v[VAL_NFG] = 1.f;
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
            {   // centre Huber loss (delta 3) on the distance
                float d2 = 0.f;
#pragma unroll
                for (int i = 0; i < 3; ++i) { const float dv = (cgt[i] - ref[i]) - ctr[i]; d2 += dv * dv; }
                v[A_CENTER] = huber(sqrtf(d2), 3.f);
            }
            int h_arg = 0, s_arg = 0;
            {   // heading class CE + residual Huber (delta 1)
                float mx;
                const float sum = softmax_denom(hs, NH, mx);
                v[A_HCLS] = -(hs[hc] - mx - logf(sum));
                float best = -1.f;
                for (int i = 0; i < NH; ++i) {
                    const float p = expf(hs[i] - mx) / sum;
                    if (p > best) { best = p; h_arg = i; }
                }
                v[A_HACC] = h_arg == hc ? 1.f : 0.f;
                v[A_HRES] = huber(fabsf(hr[hc] - hres_lab), 1.f);
            }
            {   // size class CE + residual Huber (delta 1) on the norm
                float mx;
                const float sum = softmax_denom(ss, NS, mx);
                v[A_SCLS] = -(ss[sc] - mx - logf(sum));
                float best = -1.f;
                for (int i = 0; i < NS; ++i) {
                    const float p = expf(ss[i] - mx) / sum;
                    if (p > best) { best = p; s_arg = i; }
                }
                v[A_SACC] = s_arg == sc ? 1.f : 0.f;
                float d2 = 0.f;
#pragma unroll
                for (int i = 0; i < 3; ++i) { const float dv = (sgt[i] - ex[i]) / ex[i] - sr[sc * 3 + i]; d2 += dv * dv; }
                v[A_SRES] = huber(sqrtf(d2), 1.f);
            }
            {   // corner loss: predicted box with the GT classes against the GT box and its flip
                const float cp[3] = {ref[0] + ctr[0], ref[1] + ctr[1], ref[2] + ctr[2]};
                const float ang = angle_decode(hc, hr[hc], apc);
                float sz[3];
#pragma unroll
                for (int i = 0; i < 3; ++i) sz[i] = sr[sc * 3 + i] * ex[i] + ex[i];
                float P[24], G[24], F[24];
                corners_of(cp, ang, sz, P);
                corners_of(cgt, hgt, sgt, G);
                corners_of(cgt, hgt + LOSS_PI, sgt, F);
                float dg = 0.f, df = 0.f;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    float a2 = 0.f, b2 = 0.f;
#pragma unroll
                    for (int k = 0; k < 3; ++k) {
                        const float x = P[3 * j + k] - G[3 * j + k], y = P[3 * j + k] - F[3 * j + k];
                        a2 += x * x; b2 += y * y;
                    }
                    dg += sqrtf(a2); df += sqrtf(b2);
                }
                v[A_CORNER] = huber(fminf(dg * 0.125f, df * 0.125f), 1.f);
                // IoU metrics: predicted box with the PREDICTED classes (det_base.py:488-500)
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
    // fixed-order CTA reduction: xor butterfly within each warp, then the warps in index order
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < VAL_SLOT; ++i) {
        float x = v[i];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
        if (lane == 0) s_warp[warp][i] = x;
    }
    __syncthreads();
    if (threadIdx.x < VAL_SLOT) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < VAL_THREADS / 32; ++w) s += s_warp[w][threadIdx.x];
        a.partials[(size_t)blockIdx.x * VAL_SLOT + threadIdx.x] = s;
    }
}

// One row [14 values, B, nfg, nkeep, 0] at row index state[0]++ (one thread).  The first row without a foreground row
// is recorded (the reference asserts there); rows at or past `capacity` are counted, flagged and not written.
__device__ __forceinline__ void append_row(const float *vals, int B, float nfg_raw, float nkeep_raw, float *table,
                                           int capacity, int32_t *state) {
    const int row = atomicAdd(&state[0], 1);
    if (nfg_raw == 0.f && !(state[1] & FCN_VAL_NO_FG)) {
        state[2] = row;
        state[1] |= FCN_VAL_NO_FG;
    }
    if (row >= capacity) {
        state[1] |= FCN_VAL_OVERFLOW;
        return;
    }
    float *dst = table + (size_t)row * FCN_VAL_ROW;
#pragma unroll
    for (int i = 0; i < FCN_VAL_VALUES; ++i) dst[i] = vals[i];
    dst[FCN_VAL_VALUES + 0] = (float)B;
    dst[FCN_VAL_VALUES + 1] = nfg_raw;
    dst[FCN_VAL_VALUES + 2] = nkeep_raw;
    dst[FCN_VAL_VALUES + 3] = 0.f;
}

__global__ void val_final_kernel(const __grid_constant__ fcn_val_batch_args a, int nblk) {
    __shared__ float acc[VAL_SLOT];
    if (threadIdx.x < VAL_SLOT) {
        float s = 0.f;
        for (int k = 0; k < nblk; ++k) s += a.partials[(size_t)k * VAL_SLOT + threadIdx.x];
        acc[threadIdx.x] = s;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    const float nfg_raw = acc[VAL_NFG], nkeep_raw = acc[VAL_NKEEP];
    float out[FCN_VAL_VALUES];
    loss_final_values(a, acc, nfg_raw, nkeep_raw, out);
    append_row(out, a.B, nfg_raw, nkeep_raw, a.table, a.capacity, a.state);
}

// fcn_train_states_append: `loss` is fcn_det_loss's result block (14 values, nfg, nkeep), read as it stands
__global__ void train_states_append_kernel(const float *__restrict__ loss, int B, float *__restrict__ table,
                                           int capacity, int32_t *__restrict__ state) {
    append_row(loss, B, loss[FCN_VAL_VALUES], loss[FCN_VAL_VALUES + 1], table, capacity, state);
}

// AverageMeter.update (utils/utils.py:62-66) in float64, every product and sum rounded on its own as Python does
__global__ void val_finalize_kernel(const float *__restrict__ table, int capacity, const int32_t *__restrict__ state,
                                    fcn_val_result *__restrict__ res) {
    const int k = threadIdx.x;
    const int n_rows = min(state[0], capacity);
    if (k < FCN_VAL_VALUES) {
        double sum = 0.0, count = 1e-14;
        for (int r = 0; r < n_rows; ++r) {
            const double n = (double)table[(size_t)r * FCN_VAL_ROW + FCN_VAL_VALUES];
            sum = __dadd_rn(sum, __dmul_rn((double)table[(size_t)r * FCN_VAL_ROW + k], n));
            count = __dadd_rn(count, n);
        }
        res->sum[k] = sum;
        res->avg[k] = __ddiv_rn(sum, count);
        if (k == 0) res->count = count;
    }
    if (k == 0) {
        res->rows = n_rows;
        res->added = state[0];
        res->status = state[1];
        res->first_no_fg = (state[1] & FCN_VAL_NO_FG) ? state[2] : -1;
    }
}

}  // namespace fcn

using namespace fcn;

extern "C" long long fcn_val_partials_floats(int B, int T2) {
    if (B < 1 || T2 < 1) return -1;
    return (long long)ceil_div(B * T2, VAL_THREADS) * VAL_SLOT;
}

extern "C" int fcn_val_batch(const fcn_val_batch_args *args, fcn_stream_t stream) {
    FCN_REQUIRE(args != nullptr, "args is NULL");
    const fcn_val_batch_args &a = *args;
    FCN_REQUIRE(a.B >= 1 && a.T2 >= 1 && a.NH >= 1 && a.NH <= LOSS_MAX_BINS && a.NS >= 1 && a.NS <= LOSS_MAX_BINS,
                "bad sizes");
    FCN_REQUIRE((long long)a.B * a.T2 < (1LL << 24), "B * T2 must be below 2^24 (exact float counts)");
    FCN_REQUIRE(a.logit_pitch >= a.T2, "logit_pitch must be >= T2");
    FCN_REQUIRE(a.ld_logit >= 2 + 3 + 2 * a.NH + 4 * a.NS, "ld_logit is smaller than 2 + 3 + 2*NH + 4*NS");
    FCN_REQUIRE(a.capacity >= 0, "capacity must be >= 0");
    FCN_REQUIRE(a.logits && a.center_ref2 && a.cls_label && a.size_class && a.box3d_center && a.box3d_heading &&
                    a.box3d_size && a.mean_size && a.partials && a.state && (a.table || a.capacity == 0),
                "NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int nblk = ceil_div(a.B * a.T2, VAL_THREADS);
    val_rows_kernel<<<nblk, VAL_THREADS, 0, st>>>(a);
    FCN_LAUNCH_CHECK();
    val_final_kernel<<<1, 32, 0, st>>>(a, nblk);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

extern "C" int fcn_train_states_append(const float *loss, int B, float *table, int capacity, int32_t *state,
                                       fcn_stream_t stream) {
    FCN_REQUIRE(loss != nullptr && table != nullptr && state != nullptr, "NULL pointer");
    FCN_REQUIRE(capacity >= 1, "capacity must be >= 1");
    FCN_REQUIRE(B >= 1, "B must be >= 1");
    train_states_append_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(loss, B, table, capacity, state);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

extern "C" int fcn_val_finalize(const float *table, int capacity, const int32_t *state, fcn_val_result *result,
                                fcn_stream_t stream) {
    FCN_REQUIRE(capacity >= 0, "capacity must be >= 0");
    FCN_REQUIRE(state != nullptr && result != nullptr && (table != nullptr || capacity == 0), "NULL pointer");
    val_finalize_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(table, capacity, state, result);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}
