// Training-mode kernels of the frustum hot path (config 5: cfgs/refine_car.yaml, fwd + bwd + optimizer).
//
// Replaces, for PointNetDet in train() mode, what the reference runs through PyTorch/cuDNN autograd:
//   conv (1x1 / k3 / strided / transposed) + BatchNorm with BATCH statistics + ReLU      models/common.py:38-63
//   PointNetModule / PointNetFeat (mask, max over K)                                      models/det_base.py:62-159
//   ConvFeatNet (concats, crops) and the two heads                                        models/det_base.py:163-224,367-368
//   the optimizer step (Adam or SGD)                                                      train/train_net_det.py:121-128,321-328
// Batch-statistics BN breaks the eval fusions (the statistics of layer l must be complete before layer l+1 can
// normalise its input), so the train step is a sequence of table-driven kernels over dense position-major fp32
// tensors [rows, channels]:
//   * no post-activation tensor is ever materialised: every consumer applies "scale*y + shift, ReLU" of its
//     producer (scale/shift derived on the fly from the producer's Sum(y), Sum(y^2)) while loading its operand;
//     kernel taps / strides / concats / the pixel shuffle of transposed convs / the crop are index maps of the
//     operand load (fcn_train_src / fcn_train_seg);
//   * forward GEMM  : Y = act(X) * W (+bias), epilogue accumulates Sum(y), Sum(y^2) per channel (fp64 atomics);
//   * backward       : with dz = dA * 1[pre > 0], xh = (y - mean) * invstd, the BN backward
//                       dY = scale * (dz - mean(dz) - xh * mean(dz * xh))
//                      is also applied on the fly: a column reduction produces Sum(dz), Sum(dz*xh) (= dbeta,
//                      dgamma), then  dW += act(X)^T * dY  and  dX += dY * W^T  read Y, dA and the sums directly;
//   * weights and gradients are addressed IN THE PARAMETER LAYOUT (Conv1d (Co,Ci,k), ConvTranspose1d (Ci,Co,k),
//     Conv2d (Co,Ci,1,1)) through strides, so gradients land directly in one flat bucket (one all-reduce);
//   * fp32 FMA arithmetic (parity with the fp32 reference fixture: losses 2e-4, gradients 2e-3).
#include <algorithm>
#include <type_traits>

#include "common.cuh"

namespace fcn {

constexpr float TR_EPS = 1e-5f;
constexpr int TG_BM = 64, TG_BN = 64, TG_BK = 16, TG_THREADS = 256;

struct BnCoef {
    float scale, shift, mean, invstd;
};

// scale/shift/mean/invstd of channel c of a BN layer from its Sum(y), Sum(y^2) (biased variance: training forward)
__device__ __forceinline__ BnCoef bn_coef(const double *sums, const float *gamma, const float *beta, int C, int c,
                                          double inv_count) {
    const double mean = sums[c] * inv_count;
    double var = sums[C + c] * inv_count - mean * mean;
    var = var > 0.0 ? var : 0.0;
    BnCoef r;
    r.mean = (float)mean;
    r.invstd = (float)(1.0 / sqrt(var + (double)TR_EPS));
    r.scale = gamma[c] * r.invstd;
    r.shift = beta[c] - r.mean * r.scale;
    return r;
}

// (scale, shift) with which a consumer applies source `s`'s BN to its channel c: identity without statistics or for a
// channel past the segment (!in_range)
__device__ __forceinline__ float2 src_coef(const fcn_train_src &s, int c, bool in_range) {
    if (s.sums == nullptr || !in_range) return make_float2(1.f, 0.f);
    const BnCoef b = bn_coef(s.sums, s.gamma, s.beta, s.Cstat, (s.coff + c) % s.Cstat, 1.0 / s.count);
    return make_float2(b.scale, b.shift);
}

// the producer's BN + ReLU applied to a raw element of source `s` (raw value without statistics)
__device__ __forceinline__ float src_bn_relu(const fcn_train_src &s, float x, float scale, float shift) {
    if (s.sums != nullptr) {
        x = fmaf(x, scale, shift);
        if (s.relu) x = fmaxf(x, 0.f);
    }
    return x;
}

// operand element: post-activation value of source `s` at (frustum b, position p, channel c); 0 outside [0, T*up)
__device__ __forceinline__ float src_act(const fcn_train_src &s, int b, int p, int c, float scale, float shift) {
    if (p < 0 || p >= s.T * s.up) return 0.f;
    const int row = b * s.T + p / s.up, col = s.c0 + (p % s.up) * s.cup + c;
    return src_bn_relu(s, s.raw[(size_t)row * s.ld + col], scale, shift);
}

// gradient element dY(r, n) of a layer (BN backward applied on the fly; plain layers: dY = dA).  Output column n's
// coefficients: BN scale / shift / mean / invstd and m1 = mean(dz), m2 = mean(dz * xh); identity without BN.
struct DyCoef {
    float scale, shift, mean, invstd, m1, m2;
};
__device__ __forceinline__ DyCoef dy_coef(const fcn_train_layer &L, int n) {
    DyCoef c;
    if (!L.has_bn) { c.scale = 1.f; c.m1 = c.m2 = c.mean = c.shift = 0.f; c.invstd = 1.f; return c; }
    const int co = n % L.Cout;
    const double inv = 1.0 / ((double)L.B * L.T_out * L.up);
    const BnCoef b = bn_coef(L.sums, L.gamma, L.beta, L.Cout, co, inv);
    c.scale = b.scale; c.shift = b.shift; c.mean = b.mean; c.invstd = b.invstd;
    c.m1 = (float)(L.dsums[co] * inv);
    c.m2 = (float)(L.dsums[L.Cout + co] * inv);
    return c;
}
__device__ __forceinline__ float dy_apply(const DyCoef &c, float da, float y, bool relu) {
    const float dz = (relu && fmaf(y, c.scale, c.shift) <= 0.f) ? 0.f : da;
    return c.scale * (dz - c.m1 - (y - c.mean) * c.invstd * c.m2);
}
// no BN: dA itself (dy_apply with identity coefficients would turn an inf / NaN in Y into NaN)
__device__ __forceinline__ float dy_elem(const fcn_train_layer &L, const DyCoef &c, int r, int n) {
    const float da = L.dA[(size_t)r * L.N + n];
    if (!L.has_bn) return da;
    return dy_apply(c, da, L.Y[(size_t)r * L.N + n], L.relu);
}

// one TG_BK step of the generic kernels' 4 x 4 micro-tile (rows ty*4.., columns tx*4..)
__device__ __forceinline__ void tile_fma_4x4(float (&acc)[4][4], const float (&As)[TG_BK][TG_BM + 4],
                                             const float (&Bs)[TG_BK][TG_BN + 4], int tx, int ty) {
#pragma unroll
    for (int kk = 0; kk < TG_BK; ++kk) {
        float a[4], bq[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
        for (int j = 0; j < 4; ++j) bq[j] = Bs[kk][tx * 4 + j];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bq[j], acc[i][j]);
    }
}

// Block = 32 columns (nl) x 8 row lanes (rl): each column's two partial sums a1, a2 added over the lanes in lane
// order.  Every thread calls it (barrier).  Returns `lead` (a thread of lane 0); where true, a1 and a2 hold the sums.
__device__ __forceinline__ bool column_pair_sum(float &a1, float &a2, int nl, int rl, bool lead) {
    __shared__ float s1[8][33], s2[8][33];
    s1[rl][nl] = a1; s2[rl][nl] = a2;
    __syncthreads();
    if (lead) {
        a1 = a2 = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) { a1 += s1[i][nl]; a2 += s2[i][nl]; }
    }
    return lead;
}

// weight element (segment channel c, output column n) in the parameter layout
__device__ __forceinline__ size_t w_index(const fcn_train_layer &L, const fcn_train_seg &g, int c, int n) {
    const int j = n / L.Cout, co = n - j * L.Cout;
    return (size_t)g.w_off + (size_t)c * g.s_ci + (size_t)co * L.s_co + (size_t)j * L.s_j;
}

// ------------------------------------------------------------------ forward GEMM + statistics
// The FCN layers of the refinement stage are SKINNY (M = B*T = 96..640 rows, K up to 1536): a (M/64, N/64) grid
// is 4-32 CTAs, each with a long serial K loop.  The K tiles of all segments
// are therefore linearised and split over gridDim.z; slices write partial sums to a workspace and
// train_fwd_finish_kernel adds them in a fixed order (deterministic), adds the bias, stores Y and accumulates
// the batch statistics.  gridDim.z == 1 stores Y / statistics directly.

// the CTA's 64 x 64 output tile over the linear K tiles [q_lo, q_hi) of all segments
__device__ __forceinline__ void fwd_k_tiles(const fcn_train_layer &L, int tid, int tx, int ty, int M, int r0, int n0,
                                            int q_lo, int q_hi, float (&acc)[4][4], float (&As)[TG_BK][TG_BM + 4],
                                            float (&Bs)[TG_BK][TG_BN + 4], float (&s_scale)[TG_BK],
                                            float (&s_shift)[TG_BK]) {
    int q0 = 0;                                              // first linear K tile of the current segment
    for (int sg = 0; sg < L.n_seg; ++sg) {
        const fcn_train_seg &g = L.seg[sg];
        const fcn_train_src &s = g.src;
        const double inv = s.sums != nullptr ? 1.0 / s.count : 0.0;
        const int nt = (g.C + TG_BK - 1) / TG_BK;
        const int t_lo = max(q_lo - q0, 0), t_hi = min(q_hi - q0, nt);
        q0 += nt;
        for (int t = t_lo; t < t_hi; ++t) {
            const int k0 = t * TG_BK;
            __syncthreads();
            if (tid < TG_BK) {          // src_coef, with the inverse count hoisted out of the tile loop
                const int c = k0 + tid;
                float sc = 1.f, sh = 0.f;
                if (s.sums != nullptr && c < g.C) {
                    const BnCoef b = bn_coef(s.sums, s.gamma, s.beta, s.Cstat, (s.coff + c) % s.Cstat, inv);
                    sc = b.scale; sh = b.shift;
                }
                s_scale[tid] = sc; s_shift[tid] = sh;
            }
            __syncthreads();
            // A tile: 64 rows x 16 channels (consecutive threads -> consecutive channels)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int rr = ty + 16 * i, r = r0 + rr, c = k0 + tx;
                float v = 0.f;
                if (r < M && c < g.C) {
                    const int b = r / L.T_out, tt = r - b * L.T_out;
                    v = src_act(s, b, tt * g.stride + g.tap, c, s_scale[tx], s_shift[tx]);
                }
                As[tx][rr] = v;
            }
            // B tile: 16 channels x 64 columns
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int kk = tid / 64 + 4 * i, nn = tid % 64, c = k0 + kk, n = n0 + nn;
                Bs[kk][nn] = (c < g.C && n < L.N) ? L.W[w_index(L, g, c, n)] : 0.f;
            }
            __syncthreads();
            tile_fma_4x4(acc, As, Bs, tx, ty);
        }
    }
}

// the tile's partial sums of K slice blockIdx.z: partial[z][M][N]
__device__ __forceinline__ void fwd_store_partial(const fcn_train_layer &L, int M, int r0, int n0, float *partial,
                                                  const float (&acc)[4][4]) {
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    float *dst = partial + (size_t)blockIdx.z * M * L.N;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = r0 + ty * 4 + i;
        if (r >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n < L.N) dst[(size_t)r * L.N + n] = acc[i][j];
        }
    }
}

// Generic forward.  gridDim.z > 1 stores the K slices' partial sums; gridDim.z == 1 stores Y (+bias) and, for a BN
// layer, this CTA's column sums Sum(y), Sum(y^2) over its 64 rows: ORDERED adds its 16 row groups in group order and
// stores them to slot blockIdx.x of `slots` [row block][2N] (plain stores), else they go to `sums` by atomics.
template <bool ORDERED>
__global__ void __launch_bounds__(TG_THREADS)
train_fwd_kernel(const __grid_constant__ fcn_train_layer L, float *__restrict__ partial, int tiles_per_slice,
                 float *__restrict__ slots) {
    __shared__ float As[TG_BK][TG_BM + 4], Bs[TG_BK][TG_BN + 4];
    __shared__ float s_scale[TG_BK], s_shift[TG_BK];
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    const int r0 = blockIdx.x * TG_BM, n0 = blockIdx.y * TG_BN;
    const int M = L.B * L.T_out;
    const int q_lo = blockIdx.z * tiles_per_slice, q_hi = q_lo + tiles_per_slice;
    float acc[4][4] = {};
    fwd_k_tiles(L, tid, tx, ty, M, r0, n0, q_lo, q_hi, acc, As, Bs, s_scale, s_shift);
    if (gridDim.z > 1) {
        fwd_store_partial(L, M, r0, n0, partial, acc);
        return;
    }
    if constexpr (ORDERED) {
        __shared__ float s_ps[16][TG_BN + 1], s_pq[16][TG_BN + 1];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            float ps = 0.f, pq = 0.f;
            if (n < L.N) {
                const float bias = L.bias != nullptr ? L.bias[n] : 0.f;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int r = r0 + ty * 4 + i;
                    if (r < M) {
                        const float y = acc[i][j] + bias;
                        L.Y[(size_t)r * L.N + n] = y;
                        ps += y; pq += y * y;
                    }
                }
            }
            s_ps[ty][tx * 4 + j] = ps; s_pq[ty][tx * 4 + j] = pq;
        }
        if (!L.has_bn) return;
        __syncthreads();
        if (tid < TG_BN && n0 + tid < L.N) {
            float a1 = 0.f, a2 = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) { a1 += s_ps[i][tid]; a2 += s_pq[i][tid]; }
            float *slot = slots + (size_t)blockIdx.x * 2 * L.N;
            slot[n0 + tid] = a1;
            slot[L.N + n0 + tid] = a2;
        }
    } else {
        __shared__ float s_sum[TG_BN], s_sq[TG_BN];
        if (tid < TG_BN) { s_sum[tid] = 0.f; s_sq[tid] = 0.f; }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            float ps = 0.f, pq = 0.f;
            if (n < L.N) {
                const float bias = L.bias != nullptr ? L.bias[n] : 0.f;
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int r = r0 + ty * 4 + i;
                    if (r < M) {
                        const float y = acc[i][j] + bias;
                        L.Y[(size_t)r * L.N + n] = y;
                        ps += y; pq += y * y;
                    }
                }
                if (L.has_bn) { atomicAdd(&s_sum[tx * 4 + j], ps); atomicAdd(&s_sq[tx * 4 + j], pq); }
            }
        }
        if (L.has_bn) {
            __syncthreads();
            if (tid < TG_BN && n0 + tid < L.N) {
                const int co = (n0 + tid) % L.Cout;
                atomicAdd(&L.sums[co], (double)s_sum[tid]);
                atomicAdd(&L.sums[L.Cout + co], (double)s_sq[tid]);
            }
        }
    }
}

// Y = sum over K slices (fixed order) + bias for column n, rows rb + rl, rb + rl + 8, ... < re; a1, a2 = Sum(y), Sum(y^2)
// over those rows
__device__ __forceinline__ void fwd_finish_rows(const fcn_train_layer &L, int M, const float *partial, int nslice,
                                                int n, int rl, int rb, int re, float &a1, float &a2) {
    if (n < L.N) {
        const float bias = L.bias != nullptr ? L.bias[n] : 0.f;
        for (int r = rb + rl; r < re; r += 8) {
            float y = bias;
            for (int z = 0; z < nslice; ++z) y += partial[((size_t)z * M + r) * L.N + n];
            L.Y[(size_t)r * L.N + n] = y;
            a1 += y; a2 += y * y;
        }
    }
}

// Y = sum over K slices (fixed order) + bias; batch statistics of row block blockIdx.y: to its slot [row block][2N]
// with plain stores (ORDERED), else to `sums` by atomics.  Block = 32 columns x 8 row lanes.
template <bool ORDERED>
__global__ void __launch_bounds__(256)
train_fwd_finish_kernel(const __grid_constant__ fcn_train_layer L, const float *__restrict__ partial, int nslice,
                        int rows_per_block, float *__restrict__ slots) {
    const int nl = threadIdx.x % 32, rl = threadIdx.x / 32;
    const int n = blockIdx.x * 32 + nl;
    const int M = L.B * L.T_out;
    const int rb = blockIdx.y * rows_per_block, re = min(M, rb + rows_per_block);
    float a1 = 0.f, a2 = 0.f;
    fwd_finish_rows(L, M, partial, nslice, n, rl, rb, re, a1, a2);
    if (!L.has_bn) return;
    if (column_pair_sum(a1, a2, nl, rl, rl == 0 && n < L.N)) {
        if constexpr (ORDERED) {
            float *slot = slots + (size_t)blockIdx.y * 2 * L.N;
            slot[n] = a1;
            slot[L.N + n] = a2;
        } else {
            const int co = n % L.Cout;
            atomicAdd(&L.sums[co], (double)a1);
            atomicAdd(&L.sums[L.Cout + co], (double)a2);
        }
    }
}

// Adds the slots [nrb][halves * N] of a deterministic column reduction into dst (fp64, accumulating):
//   dst[h*C + c] += sum over row blocks rb and column groups j of slots[rb][h*N + j*C + c]     (h < halves)
// (C = Cout: the up > 1 columns n = j*Cout + co of a transposed conv share channel co).  Block = 32 outputs x 8
// lanes; lane l adds the row blocks l, l + 8, ... in order, then the lanes are added in lane order: a fixed order.
__global__ void __launch_bounds__(256)
train_slots_sum_kernel(double *__restrict__ dst, const float *__restrict__ slots, int nrb, int N, int C, int halves) {
    __shared__ double s[8][33];
    const int nl = threadIdx.x % 32, rl = threadIdx.x / 32;
    const int o = blockIdx.x * 32 + nl;
    double a = 0.0;
    if (o < halves * C) {
        const int h = o / C, c = o - h * C;
        const float *col = slots + (size_t)h * N + c;
        for (int rb = rl; rb < nrb; rb += 8) {
            const float *row = col + (size_t)rb * halves * N;
            for (int j = 0; j < N; j += C) a += (double)row[j];
        }
    }
    s[rl][nl] = a;
    __syncthreads();
    if (rl == 0 && o < halves * C) {
        double t = 0.0;
#pragma unroll
        for (int i = 0; i < 8; ++i) t += s[i][nl];
        dst[o] += t;
    }
}

// ------------------------------------------------------------------ backward: column reduction Sum(dz), Sum(dz*xh)
// column n's sums over rows rb + rl, rb + rl + 8, ... < re
__device__ __forceinline__ void reduce_rows(const fcn_train_layer &L, int M, int n, int rl, int rb, int re,
                                            float &a1, float &a2) {
    if (n < L.N) {
        BnCoef b = {1.f, 0.f, 0.f, 1.f};
        if (L.has_bn) b = bn_coef(L.sums, L.gamma, L.beta, L.Cout, n % L.Cout, 1.0 / ((double)M * L.up));
        for (int r = rb + rl; r < re; r += 8) {
            const float da = L.dA[(size_t)r * L.N + n];
            if (!L.has_bn) { a1 += da; continue; }
            const float y = L.Y[(size_t)r * L.N + n];
            const float dz = (L.relu && fmaf(y, b.scale, b.shift) <= 0.f) ? 0.f : da;
            a1 += dz;
            a2 += dz * ((y - b.mean) * b.invstd);
        }
    }
}

// Sum(dz), Sum(dz*xh) of row block blockIdx.y (Sum(dA) without BN): to its slot [row block][h*N] (h = 2 with BN, 1
// without) with plain stores (ORDERED), else to `dsums` by atomics.  Block = 32 columns x 8 row lanes.
template <bool ORDERED>
__global__ void __launch_bounds__(256)
train_reduce_kernel(const __grid_constant__ fcn_train_layer L, int rows_per_block, float *__restrict__ slots) {
    const int nl = threadIdx.x % 32, rl = threadIdx.x / 32;
    const int n = blockIdx.x * 32 + nl;
    const int M = L.B * L.T_out;
    const int rb = blockIdx.y * rows_per_block, re = min(M, rb + rows_per_block);
    float a1 = 0.f, a2 = 0.f;
    reduce_rows(L, M, n, rl, rb, re, a1, a2);
    if (column_pair_sum(a1, a2, nl, rl, rl == 0 && n < L.N)) {
        if constexpr (ORDERED) {
            float *slot = slots + (size_t)blockIdx.y * (L.has_bn ? 2 : 1) * L.N;
            slot[n] = a1;
            if (L.has_bn) slot[L.N + n] = a2;
        } else {
            const int co = L.has_bn ? n % L.Cout : n;
            const int C = L.has_bn ? L.Cout : L.N;
            atomicAdd(&L.dsums[co], (double)a1);
            if (L.has_bn) atomicAdd(&L.dsums[C + co], (double)a2);
        }
    }
}

// ------------------------------------------------------------------ backward: dW += act(X)^T * dY
// the CTA's 64 channels x 64 columns tile of act(X)^T * dY over rows [rb, re) of segment g
__device__ __forceinline__ void dw_tile(const fcn_train_layer &L, const fcn_train_seg &g, int rb, int re,
                                        float (&acc)[4][4], float (&As)[TG_BK][TG_BM + 4],
                                        float (&Bs)[TG_BK][TG_BN + 4], float (&s_scale)[TG_BM],
                                        float (&s_shift)[TG_BM], DyCoef (&s_dy)[TG_BN]) {
    const fcn_train_src &s = g.src;
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    const int c0 = blockIdx.x * TG_BM, n0 = blockIdx.y * TG_BN;
    if (tid < TG_BM) {
        const float2 k = src_coef(s, c0 + tid, c0 + tid < g.C);
        s_scale[tid] = k.x; s_shift[tid] = k.y;
    }
    if (tid < TG_BN) s_dy[tid] = dy_coef(L, min(n0 + tid, L.N - 1));
    for (int rr0 = rb; rr0 < re; rr0 += TG_BK) {
        __syncthreads();
        // A tile: 16 rows x 64 channels of this segment
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int rr = tid / 64 + 4 * i, cc = tid % 64, r = rr0 + rr, c = c0 + cc;
            float v = 0.f;
            if (r < re && c < g.C) {
                const int b = r / L.T_out, t = r - b * L.T_out;
                v = src_act(s, b, t * g.stride + g.tap, c, s_scale[cc], s_shift[cc]);
            }
            As[rr][cc] = v;
        }
        // dY tile: 16 rows x 64 columns
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int rr = tid / 64 + 4 * i, nn = tid % 64, r = rr0 + rr, n = n0 + nn;
            Bs[rr][nn] = (r < re && n < L.N) ? dy_elem(L, s_dy[nn], r, n) : 0.f;
        }
        __syncthreads();
        tile_fma_4x4(acc, As, Bs, tx, ty);
    }
}

// dW tile of row slice blockIdx.z: to part[z][C][N] with plain stores (ORDERED; train_dw_sum_kernel adds the
// slices), else added to dW by atomics
template <bool ORDERED>
__global__ void __launch_bounds__(TG_THREADS)
train_dw_kernel(const __grid_constant__ fcn_train_layer L, int seg_idx, int rows_per_block, float *__restrict__ part) {
    __shared__ float As[TG_BK][TG_BM + 4], Bs[TG_BK][TG_BN + 4];   // As[row][k-channel], Bs[row][n]
    __shared__ float s_scale[TG_BM], s_shift[TG_BM];
    __shared__ DyCoef s_dy[TG_BN];
    const fcn_train_seg &g = L.seg[seg_idx];
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    const int c0 = blockIdx.x * TG_BM, n0 = blockIdx.y * TG_BN;
    const int M = L.B * L.T_out;
    const int rb = blockIdx.z * rows_per_block, re = min(M, rb + rows_per_block);
    float acc[4][4] = {};
    dw_tile(L, g, rb, re, acc, As, Bs, s_scale, s_shift, s_dy);
    float *dst = part + (size_t)blockIdx.z * g.C * L.N;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int c = c0 + ty * 4 + i;
        if (c >= g.C) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n < L.N) {
                if constexpr (ORDERED) dst[(size_t)c * L.N + n] = acc[i][j];
                else atomicAdd(&L.dW[w_index(L, g, c, n)], acc[i][j]);
            }
        }
    }
}

// dW (parameter layout) += the sum over the nz row slices, in slice order, of the partial tiles in `part`:
// [z][C][N] (generic kernel) or [z][N][C] (plain kernel, cn_layout = 0).  One read-add-store per weight: w_index is
// injective within a segment and the segments of a layer run one after another.
__global__ void train_dw_sum_kernel(const __grid_constant__ fcn_train_layer L, int seg_idx, const float *__restrict__ part,
                                    int nz, int cn_layout) {
    const fcn_train_seg &g = L.seg[seg_idx];
    const size_t total = (size_t)g.C * L.N, i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c = cn_layout ? (int)(i / L.N) : (int)(i % g.C), n = cn_layout ? (int)(i % L.N) : (int)(i / g.C);
    float sum = 0.f;
    for (int z = 0; z < nz; ++z) sum += part[(size_t)z * total + i];
    float *w = L.dW + w_index(L, g, c, n);
    *w += sum;
}

// ------------------------------------------------------------------ backward: dX(seg) += dY * W^T
// the CTA's 64 rows x 64 channels tile of dY * W^T over the columns [n_lo, n_hi) of segment g
__device__ __forceinline__ void dx_tile(const fcn_train_layer &L, const fcn_train_seg &g, int M, int r0, int c0,
                                        int n_lo, int n_hi, float (&acc)[4][4], float (&As)[TG_BK][TG_BM + 4],
                                        float (&Bs)[TG_BK][TG_BN + 4], DyCoef (&s_dy)[TG_BK]) {
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    for (int nn0 = n_lo; nn0 < n_hi; nn0 += TG_BK) {
        __syncthreads();
        if (tid < TG_BK) s_dy[tid] = dy_coef(L, min(nn0 + tid, L.N - 1));
        __syncthreads();
#pragma unroll
        for (int i = 0; i < 4; ++i) {       // dY tile: 64 rows x 16 columns (consecutive threads -> consecutive n)
            const int rr = ty + 16 * i, r = r0 + rr, n = nn0 + tx;
            As[tx][rr] = (r < M && n < n_hi) ? dy_elem(L, s_dy[tx], r, n) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {       // W tile: 16 columns x 64 channels
            const int kk = tid / 64 + 4 * i, cc = tid % 64, n = nn0 + kk, c = c0 + cc;
            Bs[kk][cc] = (n < n_hi && c < g.C) ? L.W[w_index(L, g, c, n)] : 0.f;
        }
        __syncthreads();
        tile_fma_4x4(acc, As, Bs, tx, ty);
    }
}

// source position of output row r through segment g (the consumer's index map); false outside [0, T*up)
__device__ __forceinline__ bool dx_target(const fcn_train_layer &L, const fcn_train_seg &g, int r, int &row,
                                          int &colb) {
    const fcn_train_src &s = g.src;
    const int b = r / L.T_out, t = r - b * L.T_out, p = t * g.stride + g.tap;
    if (p < 0 || p >= s.T * s.up) return false;
    row = b * s.T + p / s.up;
    colb = s.c0 + (p % s.up) * s.cup;
    return true;
}

// dX tile of column slice blockIdx.z: to part[z][M][C] with plain stores (ORDERED; train_dx_sum_kernel adds the
// slices), else added to src.grad through the operand's index map by atomics
template <bool ORDERED>
__global__ void __launch_bounds__(TG_THREADS)
train_dx_kernel(const __grid_constant__ fcn_train_layer L, int seg_idx, int n_per_slice, float *__restrict__ part) {
    __shared__ float As[TG_BK][TG_BM + 4], Bs[TG_BK][TG_BN + 4];   // As[n][row], Bs[n][channel]
    __shared__ DyCoef s_dy[TG_BK];
    const fcn_train_seg &g = L.seg[seg_idx];
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    const int r0 = blockIdx.x * TG_BM, c0 = blockIdx.y * TG_BN;
    const int M = L.B * L.T_out;
    float acc[4][4] = {};
    const int n_lo = blockIdx.z * n_per_slice, n_hi = min(L.N, n_lo + n_per_slice);
    dx_tile(L, g, M, r0, c0, n_lo, n_hi, acc, As, Bs, s_dy);
    if constexpr (ORDERED) {
        float *dst = part + (size_t)blockIdx.z * M * g.C;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int r = r0 + ty * 4 + i;
            if (r >= M) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int c = c0 + tx * 4 + j;
                if (c < g.C) dst[(size_t)r * g.C + c] = acc[i][j];
            }
        }
    } else {
        const fcn_train_src &s = g.src;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int r = r0 + ty * 4 + i;
            if (r >= M) continue;
            int row, colb;
            if (!dx_target(L, g, r, row, colb)) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int c = c0 + tx * 4 + j;
                if (c < g.C) atomicAdd(&s.grad[(size_t)row * s.ld + colb + c], acc[i][j]);
            }
        }
    }
}

// src.grad += the sum over the nz column slices, in slice order, of part[z][M][C], through the index map of
// train_dx_kernel: one read-add-store per element (the map is injective within a segment: distinct output rows reach
// distinct source positions; the segments of a layer and the layers run one after another)
__global__ void train_dx_sum_kernel(const __grid_constant__ fcn_train_layer L, int seg_idx, const float *__restrict__ part,
                                    int nz) {
    const fcn_train_seg &g = L.seg[seg_idx];
    const int M = L.B * L.T_out;
    const size_t total = (size_t)M * g.C, i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int r = (int)(i / g.C), c = (int)(i % g.C);
    int row, colb;
    if (!dx_target(L, g, r, row, colb)) return;
    float sum = 0.f;
    for (int z = 0; z < nz; ++z) sum += part[(size_t)z * total + i];
    float *d = g.src.grad + (size_t)row * g.src.ld + colb + c;
    *d += sum;
}

// ------------------------------------------------------------------ PointNet pooling (mask, max over K) fwd / bwd
// feat[(b,t), c] = cnt>0 ? max_k relu(scale*y + shift) : 0 ; argmax kept for the backward; one-hot columns appended
__global__ void train_pool_fwd_kernel(fcn_train_pool_args P) {
    const int bt = blockIdx.x, c = blockIdx.y * blockDim.x + threadIdx.x;
    if (c >= P.C + P.V) return;
    float *out = P.feat + (size_t)bt * P.ld_feat;
    if (c >= P.C) { out[c] = P.one_hot[(size_t)(bt / P.T) * P.V + (c - P.C)]; return; }
    const BnCoef b = bn_coef(P.sums, P.gamma, P.beta, P.C, c, 1.0 / ((double)P.B * P.T * P.K));
    float best = -INFINITY;
    int arg = 0;
    const float *y = P.Y + (size_t)bt * P.K * P.C + c;
    const bool valid = P.cnt[bt] > 0;
    for (int k = 0; k < P.K; ++k) {
        float a = fmaxf(fmaf(y[(size_t)k * P.C], b.scale, b.shift), 0.f);
        if (!valid) a = 0.f;                 // x * (cnt > 0)  (det_base.py:100-101): all-zero rows, argmax = 0
        if (a > best) { best = a; arg = k; }
    }
    out[c] = best;
    P.argmax[(size_t)bt * P.C + c] = arg;
}
// dA3[(b,t,argmax), c] = cnt>0 ? dfeat[(b,t), c] : 0   (dA3 is zero-filled by the caller)
__global__ void train_pool_bwd_kernel(fcn_train_pool_args P) {
    const int bt = blockIdx.x, c = blockIdx.y * blockDim.x + threadIdx.x;
    if (c >= P.C || P.cnt[bt] <= 0) return;
    const int arg = P.argmax[(size_t)bt * P.C + c];
    P.dA[((size_t)bt * P.K + arg) * P.C + c] = P.dfeat[(size_t)bt * P.ld_feat + c];
}

// ------------------------------------------------------------------ end of step: BN bookkeeping for ALL layers
// running statistics (momentum 0.1, unbiased variance; models/common.py BatchNorm defaults), dgamma / dbeta / dbias
__global__ void train_finalize_kernel(const fcn_train_layer *layers, int n_layers, int update_running) {
    const fcn_train_layer &L = layers[blockIdx.x];
    const double cnt = (double)L.B * L.T_out * L.up;
    for (int c = threadIdx.x; c < (L.has_bn ? L.Cout : L.N); c += blockDim.x) {
        if (!L.has_bn) {
            if (L.dbias != nullptr) L.dbias[c] += (float)L.dsums[c];
            continue;
        }
        L.dbeta[c] += (float)L.dsums[c];
        L.dgamma[c] += (float)L.dsums[L.Cout + c];
        if (update_running) {
            const double mean = L.sums[c] / cnt;
            double var = L.sums[L.Cout + c] / cnt - mean * mean;
            var = var > 0.0 ? var : 0.0;
            const double unb = cnt > 1.0 ? var * cnt / (cnt - 1.0) : var;
            L.run_mean[c] = (float)(0.9 * (double)L.run_mean[c] + 0.1 * mean);
            L.run_var[c] = (float)(0.9 * (double)L.run_var[c] + 0.1 * unb);
        }
    }
}

// ------------------------------------------------------------------ fused Adam over the flat parameter bucket
// torch.optim.Adam semantics (train_net_det.py:322-323): g += wd * p; m, v EMAs; bias correction; p -= lr * mhat/(sqrt(vhat)+eps)
__global__ void train_adam_kernel(float *__restrict__ p, const float *__restrict__ g, float *__restrict__ m,
                                  float *__restrict__ v, size_t n, float lr, float b1, float b2, float eps, float wd,
                                  float bc1, float bc2, float gscale) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float gi = g[i] * gscale + wd * p[i];
    const float mi = b1 * m[i] + (1.f - b1) * gi;
    const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
    m[i] = mi; v[i] = vi;
    const float denom = sqrtf(vi) / sqrtf(bc2) + eps;
    p[i] -= (lr / bc1) * (mi / denom);
}

// ------------------------------------------------------------------ fused SGD over the flat parameter bucket
// torch.optim.SGD (train_net_det.py:324-326) as torch/optim/sgd.py::_single_tensor_sgd does it, one rounding per torch
// op: d = g + wd * p (skipped at wd == 0, as torch skips it); buf = d on the first step, else buf * momentum + d;
// p += -lr * (buf or d).  torch's CUDA add(x, y, alpha) computes x + alpha * y as one FMA, so those two steps are
// __fmaf_rn; every rounding is an explicit intrinsic so that -fmad cannot change the result.
__global__ void train_sgd_kernel(float *__restrict__ p, const float *__restrict__ g, float *__restrict__ buf, size_t n,
                                 float lr, float momentum, float wd, int first, float gscale) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float pi = p[i];
    float d = __fmul_rn(g[i], gscale);
    if (wd != 0.f) d = __fmaf_rn(wd, pi, d);                             // grad.add(param, alpha=wd)
    if (momentum != 0.f) {
        if (!first) d = __fadd_rn(__fmul_rn(buf[i], momentum), d);       // buf.mul_(momentum).add_(d)
        buf[i] = d;
    }
    p[i] = __fmaf_rn(-lr, d, pi);                                        // param.add_(d, alpha=-lr)
}


// =====================================================================================================
// Fast path for the PointNet layers 2/3 (97 % of the step's FLOPs): single source, 1x1 conv, rows map 1:1
// (tap 0, stride 1, no pixel shuffle), channels and columns multiples of 64 up to 512 (host_plain states the rule).
// 128 x 64 x 16 tiles, 8 x 4 micro-tiles, float4 global loads along the contiguous axis, register prefetch of the
// next tile.  Same arithmetic (fp32 FMA, same on-the-fly BN / ReLU forward and backward) as the generic kernels above.
// =====================================================================================================
constexpr int FP_BM = 128, FP_BN = 64, FP_BK = 16, FP_THREADS = 256;

// one FP_BK step of the plain kernels' 8 x 4 micro-tile (rows ty*8.., columns tx*4..), float4 shared loads
__device__ __forceinline__ void tile_fma_8x4(float (&acc)[8][4], const float (&As)[FP_BK][FP_BM + 4],
                                             const float (&Bs)[FP_BK][FP_BN + 4], int tx, int ty) {
#pragma unroll
    for (int kk = 0; kk < FP_BK; ++kk) {
        const float4 a0 = *(const float4 *)&As[kk][ty * 8], a1 = *(const float4 *)&As[kk][ty * 8 + 4];
        const float4 b0 = *(const float4 *)&Bs[kk][tx * 4];
        const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float b[4] = {b0.x, b0.y, b0.z, b0.w};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
}

// the plain forward's 128 x 64 output tile over all of K (s_scale / s_shift: the source's BN, staged for all K)
__device__ __forceinline__ void fwd_plain_tiles(const fcn_train_layer &L, const fcn_train_seg &g, int tid, int tx,
                                                int ty, int r0, int n0, int M, int K, float (&acc)[8][4],
                                                float (&As)[FP_BK][FP_BM + 4], float (&Bs)[FP_BK][FP_BN + 4],
                                                const float (&s_scale)[512], const float (&s_shift)[512]) {
    const fcn_train_src &s = g.src;
    // A: 128 rows x 16 k = 512 float4 (2 per thread); B: 64 n x 16 k = 256 float4 (1 per thread)
    const int arow = tid / 4, akq = (tid % 4) * 4;
    const int bn = tid / 4, bkq = (tid % 4) * 4;
    float4 pa[2], pb;
    auto gload = [&](int k0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = r0 + arow + 64 * h;
            pa[h] = r < M ? *(const float4 *)(s.raw + (size_t)r * s.ld + k0 + akq) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        pb = *(const float4 *)(L.W + g.w_off + (size_t)(n0 + bn) * L.s_co + k0 + bkq);
    };
    auto sstore = [&](int k0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float v[4] = {pa[h].x, pa[h].y, pa[h].z, pa[h].w};
            const bool ok = r0 + arow + 64 * h < M;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float x = src_bn_relu(s, v[i], s_scale[k0 + akq + i], s_shift[k0 + akq + i]);
                As[akq + i][arow + 64 * h] = ok ? x : 0.f;
            }
        }
        Bs[bkq + 0][bn] = pb.x; Bs[bkq + 1][bn] = pb.y; Bs[bkq + 2][bn] = pb.z; Bs[bkq + 3][bn] = pb.w;
    };
    gload(0);
    for (int k0 = 0; k0 < K; k0 += FP_BK) {
        __syncthreads();
        sstore(k0);
        __syncthreads();
        if (k0 + FP_BK < K) gload(k0 + FP_BK);
        tile_fma_8x4(acc, As, Bs, tx, ty);
    }
}

// Y[M,N] = act(X[M,K]) * W^T   (W in parameter layout (N,K): both operands contiguous along K).  This CTA's column
// sums over its 128 rows: ORDERED adds its 16 row groups in group order and stores them to slot blockIdx.x of `slots`
// [row block][2N] (plain stores), else they go to `sums` by atomics.
template <bool ORDERED>
__global__ void __launch_bounds__(FP_THREADS)
train_fwd_plain_kernel(const __grid_constant__ fcn_train_layer L, float *__restrict__ slots) {
    __shared__ __align__(16) float As[FP_BK][FP_BM + 4], Bs[FP_BK][FP_BN + 4];
    __shared__ float s_scale[512], s_shift[512];
    // column sums Sum(y), Sum(y^2): per row group (ORDERED), else one per column, zeroed before the main loop
    __shared__ std::conditional_t<ORDERED, float[16][FP_BN + 1], float[FP_BN]> s_ps, s_pq;
    const fcn_train_seg &g = L.seg[0];
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    const int r0 = blockIdx.x * FP_BM, n0 = blockIdx.y * FP_BN;
    const int M = L.B * L.T_out, K = g.C;
    for (int c = tid; c < K; c += FP_THREADS) {
        const float2 k = src_coef(g.src, c, true);
        s_scale[c] = k.x; s_shift[c] = k.y;
    }
    if constexpr (!ORDERED)
        if (tid < FP_BN) { s_ps[tid] = 0.f; s_pq[tid] = 0.f; }
    __syncthreads();
    float acc[8][4] = {};
    fwd_plain_tiles(L, g, tid, tx, ty, r0, n0, M, K, acc, As, Bs, s_scale, s_shift);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int n = n0 + tx * 4 + j;
        float ps = 0.f, pq = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = r0 + ty * 8 + i;
            if (r < M) {
                const float y = acc[i][j];
                L.Y[(size_t)r * L.N + n] = y;
                ps += y; pq += y * y;
            }
        }
        if constexpr (ORDERED) {
            s_ps[ty][tx * 4 + j] = ps; s_pq[ty][tx * 4 + j] = pq;
        } else {
            atomicAdd(&s_ps[tx * 4 + j], ps);
            atomicAdd(&s_pq[tx * 4 + j], pq);
        }
    }
    __syncthreads();
    if (tid < FP_BN) {
        if constexpr (ORDERED) {
            float a1 = 0.f, a2 = 0.f;
#pragma unroll
            for (int i = 0; i < 16; ++i) { a1 += s_ps[i][tid]; a2 += s_pq[i][tid]; }
            float *slot = slots + (size_t)blockIdx.x * 2 * L.N;
            slot[n0 + tid] = a1;
            slot[L.N + n0 + tid] = a2;
        } else {
            atomicAdd(&L.sums[n0 + tid], (double)s_ps[tid]);
            atomicAdd(&L.sums[L.Cout + n0 + tid], (double)s_pq[tid]);
        }
    }
}

// dX[M,K] += dY[M,N] * W   (W (N,K): contiguous along K).  One CTA owns each element and there is no N split, so
// the accumulation into the source gradient (shared with its other consumers) is a plain read-add-store.
__global__ void __launch_bounds__(FP_THREADS)
train_dx_plain_kernel(const __grid_constant__ fcn_train_layer L) {
    __shared__ __align__(16) float As[FP_BK][FP_BM + 4], Bs[FP_BK][FP_BN + 4];
    __shared__ DyCoef s_c[512];
    const fcn_train_seg &g = L.seg[0];
    const fcn_train_src &s = g.src;
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    const int r0 = blockIdx.x * FP_BM, c0 = blockIdx.y * FP_BN;
    const int M = L.B * L.T_out, N = L.N;
    for (int n = tid; n < N; n += FP_THREADS) s_c[n] = dy_coef(L, n);
    __syncthreads();
    const bool relu = L.relu != 0;
    const int arow = tid / 4, anq = (tid % 4) * 4;          // dY tile: 128 rows x 16 n
    const int bnr = tid / 16, bkq = (tid % 16) * 4;         // W tile: 16 n x 64 k
    float4 pda[2], py[2], pb;
    auto gload = [&](int n0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = r0 + arow + 64 * h;
            if (r < M) {
                pda[h] = *(const float4 *)(L.dA + (size_t)r * N + n0 + anq);
                py[h] = *(const float4 *)(L.Y + (size_t)r * N + n0 + anq);
            } else {
                pda[h] = py[h] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
        pb = *(const float4 *)(L.W + g.w_off + (size_t)(n0 + bnr) * L.s_co + c0 + bkq);
    };
    auto sstore = [&](int n0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const float da[4] = {pda[h].x, pda[h].y, pda[h].z, pda[h].w}, y[4] = {py[h].x, py[h].y, py[h].z, py[h].w};
            const bool ok = r0 + arow + 64 * h < M;
#pragma unroll
            for (int i = 0; i < 4; ++i)
                As[anq + i][arow + 64 * h] = ok ? dy_apply(s_c[n0 + anq + i], da[i], y[i], relu) : 0.f;
        }
        *(float4 *)&Bs[bnr][bkq] = pb;
    };
    float acc[8][4] = {};
    gload(0);
    for (int n0 = 0; n0 < N; n0 += FP_BK) {
        __syncthreads();
        sstore(n0);
        __syncthreads();
        if (n0 + FP_BK < N) gload(n0 + FP_BK);
        tile_fma_8x4(acc, As, Bs, tx, ty);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int r = r0 + ty * 8 + i;
        if (r < M) {
            float4 *dst = (float4 *)(s.grad + (size_t)r * s.ld + c0 + tx * 4);
            const float4 o = *dst;
            *dst = make_float4(o.x + acc[i][0], o.y + acc[i][1], o.z + acc[i][2], o.w + acc[i][3]);
        }
    }
}

// the plain dW's 128 columns x 64 channels tile of dY^T * act(X) over rows [rb, re)
__device__ __forceinline__ void dw_plain_tiles(const fcn_train_layer &L, const fcn_train_seg &g, int tid, int n0,
                                               int c0, int N, int rb, int re, float (&acc)[8][4],
                                               float (&As)[FP_BK][FP_BM + 4], float (&Bs)[FP_BK][FP_BN + 4],
                                               DyCoef (&s_c)[FP_BM], float (&s_scale)[FP_BN],
                                               float (&s_shift)[FP_BN]) {
    const fcn_train_src &s = g.src;
    const int tx = tid % 16, ty = tid / 16;
    if (tid < FP_BM) s_c[tid] = dy_coef(L, min(n0 + tid, N - 1));
    if (tid < FP_BN) {
        const float2 k = src_coef(s, c0 + tid, true);
        s_scale[tid] = k.x; s_shift[tid] = k.y;
    }
    __syncthreads();
    const bool relu = L.relu != 0;
    // dY tile: 16 rows x 128 n = 512 float4 (2 per thread); X tile: 16 rows x 64 k = 256 float4 (1 per thread)
    const int ar = tid / 32, anq = (tid % 32) * 4;
    const int br = tid / 16, bkq = (tid % 16) * 4;
    float4 pda[2], py[2], px;
    const bool n_ok = n0 + anq < N;      // N % 64 == 0: a 128-wide tile may hang over by 64
    auto gload = [&](int m0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = m0 + ar + 8 * h;
            if (r < re && n_ok) {
                pda[h] = *(const float4 *)(L.dA + (size_t)r * N + n0 + anq);
                py[h] = *(const float4 *)(L.Y + (size_t)r * N + n0 + anq);
            } else {
                pda[h] = py[h] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
        const int r = m0 + br;
        px = r < re ? *(const float4 *)(s.raw + (size_t)r * s.ld + c0 + bkq) : make_float4(0.f, 0.f, 0.f, 0.f);
    };
    auto sstore = [&](int m0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const bool ok = m0 + ar + 8 * h < re && n_ok;
            float4 o;
            o.x = ok ? dy_apply(s_c[anq + 0], pda[h].x, py[h].x, relu) : 0.f;
            o.y = ok ? dy_apply(s_c[anq + 1], pda[h].y, py[h].y, relu) : 0.f;
            o.z = ok ? dy_apply(s_c[anq + 2], pda[h].z, py[h].z, relu) : 0.f;
            o.w = ok ? dy_apply(s_c[anq + 3], pda[h].w, py[h].w, relu) : 0.f;
            *(float4 *)&As[ar + 8 * h][anq] = o;
        }
        const bool ok = m0 + br < re;
        float x[4] = {px.x, px.y, px.z, px.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            x[i] = src_bn_relu(s, x[i], s_scale[bkq + i], s_shift[bkq + i]);
            if (!ok) x[i] = 0.f;
        }
        *(float4 *)&Bs[br][bkq] = make_float4(x[0], x[1], x[2], x[3]);
    };
    gload(rb);
    for (int m0 = rb; m0 < re; m0 += FP_BK) {
        __syncthreads();
        sstore(m0);
        __syncthreads();
        if (m0 + FP_BK < re) gload(m0 + FP_BK);
        tile_fma_8x4(acc, As, Bs, tx, ty);
    }
}

// dW[N,K] += dY[M,N]^T * act(X[M,K])   over the row slice [z*rows_per_block, ...): to part[z][N][C] with plain
// float4 stores (ORDERED; train_dw_sum_kernel adds the slices), else atomicAdd into the bucket
template <bool ORDERED>
__global__ void __launch_bounds__(FP_THREADS)
train_dw_plain_kernel(const __grid_constant__ fcn_train_layer L, int rows_per_block, float *__restrict__ part) {
    __shared__ __align__(16) float As[FP_BK][FP_BM + 4], Bs[FP_BK][FP_BN + 4];   // As[row][n], Bs[row][k]
    __shared__ DyCoef s_c[FP_BM];
    __shared__ float s_scale[FP_BN], s_shift[FP_BN];
    const fcn_train_seg &g = L.seg[0];
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    const int n0 = blockIdx.x * FP_BM, c0 = blockIdx.y * FP_BN;
    const int M = L.B * L.T_out, N = L.N, C = g.C;
    const int rb = blockIdx.z * rows_per_block, re = min(M, rb + rows_per_block);
    float acc[8][4] = {};
    dw_plain_tiles(L, g, tid, n0, c0, N, rb, re, acc, As, Bs, s_c, s_scale, s_shift);
    float *dst = part + (size_t)blockIdx.z * N * C;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int n = n0 + ty * 8 + i;
        if (n >= N) continue;
        if constexpr (ORDERED) {
            *(float4 *)(dst + (size_t)n * C + c0 + tx * 4) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
                atomicAdd(&L.dW[g.w_off + (size_t)n * L.s_co + c0 + tx * 4 + j], acc[i][j]);
        }
    }
}

static int check_layer(const fcn_train_layer &L) {
    FCN_REQUIRE(L.B >= 1 && L.T_out >= 1 && L.N >= 1 && L.Cout >= 1 && L.up >= 1, "bad layer shape");
    FCN_REQUIRE(L.n_seg >= 1 && L.n_seg <= FCN_MAX_SEGS, "n_seg out of range");
    FCN_REQUIRE(L.W && L.Y, "NULL weight / output");
    FCN_REQUIRE(!L.has_bn || (L.sums && L.gamma && L.beta), "BN layer without statistics buffers");
    for (int i = 0; i < L.n_seg; ++i) {
        const fcn_train_src &s = L.seg[i].src;
        FCN_REQUIRE(s.raw && s.T >= 1 && s.up >= 1 && s.ld >= 1 && L.seg[i].C >= 1 && L.seg[i].stride >= 1, "bad segment");
        FCN_REQUIRE(s.sums == nullptr || (s.gamma && s.beta && s.Cstat >= 1 && s.count > 0), "bad source statistics");
    }
    return FCN_OK;
}

// the layer takes the plain kernels (shared-memory tables: C, N <= 512; float4 loads: 16-byte aligned rows)
static bool host_plain(const fcn_train_layer &L) {
    const fcn_train_seg &g = L.seg[0];
    return L.n_seg == 1 && g.tap == 0 && g.stride == 1 && g.src.up == 1 && L.up == 1 && g.src.T == L.T_out &&
           g.s_ci == 1 && g.C % 64 == 0 && g.C <= 512 && L.N % 64 == 0 && L.N <= 512 && g.src.c0 == 0 &&
           g.src.ld % 4 == 0 && g.w_off % 4 == 0 && L.s_co % 4 == 0 && L.has_bn && L.bias == nullptr &&
           L.Cout == L.N;
}

}  // namespace fcn

using namespace fcn;

// The generic kernels split their reduction until about this many CTAs exist: 2 per SM of the 148-SM GPU the splits
// were tuned for, not the H100's 132.  Kept because the forward's K split decides the order in which its partial
// sums add up, so another value changes the bits of Y.
constexpr int SPLIT_CTAS = 2 * 148;

// K slices of the generic forward GEMM for this layer (1 = no split); `workspace_floats` bounds the partial sums
static int fwd_slices(const fcn_train_layer &L, long long workspace_floats, int *tiles_per_slice) {
    const int M = L.B * L.T_out;
    int tiles = 0;
    for (int i = 0; i < L.n_seg; ++i) tiles += ceil_div(L.seg[i].C, TG_BK);
    const int ctas = ceil_div(M, TG_BM) * ceil_div(L.N, TG_BN);
    int want = ceil_div(SPLIT_CTAS, ctas);
    if (want > tiles / 2) want = tiles / 2;                  // at least two K tiles per slice
    const long long fit = workspace_floats / ((long long)M * L.N);
    if (want > fit) want = (int)fit;
    if (want < 2) { *tiles_per_slice = tiles; return 1; }
    *tiles_per_slice = ceil_div(tiles, want);
    return ceil_div(tiles, *tiles_per_slice);
}

// Rows (dW) or columns (dX) per CTA of a backward reduction of length `len` over `ctas` output tiles: about
// SPLIT_CTAS CTAs in all, a multiple of TG_BK and at least two tiles.  The layers are skinny, and a handful of CTAs
// with long serial loops would be the bottleneck (the outputs are atomic accumulations).
static int split_len(int len, int ctas) {
    const int per = ceil_div(ceil_div(len, ceil_div(SPLIT_CTAS, ctas)), TG_BK) * TG_BK;
    return per < 2 * TG_BK ? 2 * TG_BK : per;
}

// How a layer's GEMMs are split.  Both modes launch these splits.  The forward's K split is the largest that
// `fwd_workspace_floats` holds: the default forward passes its workspace, the deterministic mode and the workspace
// queries pass FWD_UNBOUNDED, so every split the deterministic mode uses depends on the layer's shape only.
constexpr long long FWD_UNBOUNDED = (long long)1 << 40;

struct TrainPlan {
    bool plain;                  // host_plain: the 128 x 64 kernels, which split neither K nor the dX columns
    int nslice, tiles_per_slice; // K slices of the generic forward and linear K tiles per slice
    long long partial;           // floats of the generic forward's K-slice partial sums (0 without a split)
    int stats_rpb;               // rows per block of the forward statistics: the plain or generic CTA's rows, or the
                                 // finish kernel's when K is split
    int reduce_rpb;              // rows per block of the backward's column reduction
    int dw_rpb[FCN_MAX_SEGS];    // per segment: rows per slice of dW
    int dx_nps[FCN_MAX_SEGS];    // per segment: columns per slice of the generic dX
};

static TrainPlan train_plan(const fcn_train_layer &L, long long fwd_workspace_floats) {
    const int M = L.B * L.T_out;
    TrainPlan p{};
    p.plain = host_plain(L);
    p.nslice = fwd_slices(L, fwd_workspace_floats, &p.tiles_per_slice);
    p.partial = p.nslice > 1 ? (long long)p.nslice * M * L.N : 0;
    p.stats_rpb = p.plain ? FP_BM : p.nslice > 1 ? 32 : TG_BM;
    p.reduce_rpb = M >= 4096 ? 256 : 32;
    for (int sg = 0; sg < L.n_seg; ++sg) {
        const int C = L.seg[sg].C;
        p.dw_rpb[sg] = p.plain ? 1024 : split_len(M, ceil_div(C, TG_BM) * ceil_div(L.N, TG_BN));
        p.dx_nps[sg] = p.plain ? 0 : split_len(L.N, ceil_div(M, TG_BM) * ceil_div(C, TG_BN));
    }
    return p;
}

static bool shape_ok(const fcn_train_layer &L) {
    if (L.B < 1 || L.T_out < 1 || L.N < 1 || L.Cout < 1 || L.up < 1 || L.n_seg < 1 || L.n_seg > FCN_MAX_SEGS)
        return false;
    for (int i = 0; i < L.n_seg; ++i)
        if (L.seg[i].C < 1) return false;
    return true;
}

// ------------------------------------------------------------------ deterministic mode
// The same GEMMs with every float atomic replaced by plain stores of partial results into the workspace and ordered
// sums of those partials: per-row-block column sums (slots) for Sum(y), Sum(y^2), Sum(dz), Sum(dz*xh), row-slice
// tiles for dW and column-slice tiles for dX.  The forward keeps its K-split partials, then the slots; the backward's
// launches use the workspace one after another.
static long long det_floats(const fcn_train_layer &L) {
    const TrainPlan p = train_plan(L, FWD_UNBOUNDED);
    const int M = L.B * L.T_out;
    const long long fwd = (p.plain ? 0 : p.partial) + (L.has_bn ? (long long)ceil_div(M, p.stats_rpb) * 2 * L.N : 0);
    long long bwd = (long long)ceil_div(M, p.reduce_rpb) * (L.has_bn ? 2 : 1) * L.N;
    for (int sg = 0; sg < L.n_seg; ++sg) {
        const int C = L.seg[sg].C;
        bwd = std::max(bwd, (long long)ceil_div(M, p.dw_rpb[sg]) * C * L.N);
        if (!p.plain) bwd = std::max(bwd, (long long)ceil_div(L.N, p.dx_nps[sg]) * M * C);
    }
    return std::max(fwd, bwd);
}

static int det_workspace_check(const fcn_train_layer &L, const float *ws, long long ws_floats) {
    FCN_REQUIRE(ws != nullptr, "NULL workspace (the deterministic kernels need fcn_train_deterministic_workspace_floats)");
    FCN_REQUIRE(ws_floats >= det_floats(L), "workspace smaller than fcn_train_deterministic_workspace_floats(layer)");
    return FCN_OK;
}

static int launch_slots_sum(double *dst, const float *slots, int nrb, int N, int C, int halves, cudaStream_t st) {
    train_slots_sum_kernel<<<ceil_div(halves * C, 32), 256, 0, st>>>(dst, slots, nrb, N, C, halves);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

// cudaGetLastError after a launch, reported as an error of the entry `fn`
static int launch_error(const char *fn) {
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? FCN_OK : cuda_fail(fn, e);
}

// Forward of one layer for the entry `fn`; `ordered` is the deterministic mode, whose statistics go to slots after
// the K-split partials.
static int train_forward(const char *fn, const fcn_train_layer *L, float *ws, long long ws_floats, bool ordered,
                         cudaStream_t st) {
    if (L == nullptr) return invalid(fn, "NULL layer");
    if (int rc = check_layer(*L)) return rc;
    if (ordered)
        if (int rc = det_workspace_check(*L, ws, ws_floats)) return rc;
    const TrainPlan p = train_plan(*L, ordered ? FWD_UNBOUNDED : ws != nullptr ? ws_floats : 0);
    const int M = L->B * L->T_out, nrb = ceil_div(M, p.stats_rpb);
    float *slots = ordered ? ws + (p.plain ? 0 : p.partial) : nullptr;
    if (p.plain) {
        dim3 grid(nrb, L->N / FP_BN);
        (ordered ? train_fwd_plain_kernel<true> : train_fwd_plain_kernel<false>)<<<grid, FP_THREADS, 0, st>>>(*L, slots);
        if (int rc = launch_error(fn)) return rc;
    } else {
        dim3 grid(ceil_div(M, TG_BM), ceil_div(L->N, TG_BN), p.nslice);
        (ordered ? train_fwd_kernel<true> : train_fwd_kernel<false>)<<<grid, TG_THREADS, 0, st>>>(
            *L, ws, p.tiles_per_slice, slots);
        if (int rc = launch_error(fn)) return rc;
        if (p.nslice > 1) {
            dim3 gf(ceil_div(L->N, 32), nrb);
            (ordered ? train_fwd_finish_kernel<true> : train_fwd_finish_kernel<false>)<<<gf, 256, 0, st>>>(
                *L, ws, p.nslice, p.stats_rpb, slots);
            if (int rc = launch_error(fn)) return rc;
        }
    }
    if (ordered && L->has_bn) return launch_slots_sum(L->sums, slots, nrb, L->N, L->Cout, 2, st);
    return FCN_OK;
}

// Backward of one layer for the entry `fn`; `ordered` is the deterministic mode, which adds every set of partials it
// stores in the workspace before its next launch.
static int train_backward(const char *fn, const fcn_train_layer *L, int need_dx_mask, float *ws, long long ws_floats,
                          bool ordered, cudaStream_t st) {
    if (L == nullptr) return invalid(fn, "NULL layer");
    if (int rc = check_layer(*L)) return rc;
    if (!(L->dA && L->dW && L->dsums)) return invalid(fn, "NULL gradient buffers");
    if (ordered)
        if (int rc = det_workspace_check(*L, ws, ws_floats)) return rc;
    const TrainPlan p = train_plan(*L, FWD_UNBOUNDED);
    const int M = L->B * L->T_out, N = L->N;
    {   // Sum(dz), Sum(dz * xh) per channel
        const int nrb = ceil_div(M, p.reduce_rpb);
        (ordered ? train_reduce_kernel<true> : train_reduce_kernel<false>)<<<dim3(ceil_div(N, 32), nrb), 256, 0, st>>>(
            *L, p.reduce_rpb, ws);
        if (int rc = launch_error(fn)) return rc;
        if (ordered)
            if (int rc = launch_slots_sum(L->dsums, ws, nrb, N, L->has_bn ? L->Cout : N, L->has_bn ? 2 : 1, st))
                return rc;
    }
    for (int sg = 0; sg < L->n_seg; ++sg) {
        const int C = L->seg[sg].C, nz = ceil_div(M, p.dw_rpb[sg]);
        if (p.plain) {
            dim3 grid(ceil_div(N, FP_BM), C / FP_BN, nz);
            (ordered ? train_dw_plain_kernel<true> : train_dw_plain_kernel<false>)<<<grid, FP_THREADS, 0, st>>>(
                *L, p.dw_rpb[sg], ws);
        } else {
            dim3 grid(ceil_div(C, TG_BM), ceil_div(N, TG_BN), nz);
            (ordered ? train_dw_kernel<true> : train_dw_kernel<false>)<<<grid, TG_THREADS, 0, st>>>(
                *L, sg, p.dw_rpb[sg], ws);
        }
        if (int rc = launch_error(fn)) return rc;
        if (ordered) {
            train_dw_sum_kernel<<<ceil_div(C * N, 256), 256, 0, st>>>(*L, sg, ws, nz, !p.plain);
            if (int rc = launch_error(fn)) return rc;
        }
        if (!((need_dx_mask >> sg) & 1) || L->seg[sg].src.grad == nullptr) continue;
        if (p.plain) {      // one CTA per element, no split: order-free in both modes
            train_dx_plain_kernel<<<dim3(ceil_div(M, FP_BM), C / FP_BN), FP_THREADS, 0, st>>>(*L);
            if (int rc = launch_error(fn)) return rc;
            continue;
        }
        const int nzx = ceil_div(N, p.dx_nps[sg]);
        (ordered ? train_dx_kernel<true> : train_dx_kernel<false>)<<<dim3(ceil_div(M, TG_BM), ceil_div(C, TG_BN), nzx),
                                                                      TG_THREADS, 0, st>>>(*L, sg, p.dx_nps[sg], ws);
        if (int rc = launch_error(fn)) return rc;
        if (ordered) {
            train_dx_sum_kernel<<<(unsigned)(((long long)M * C + 255) / 256), 256, 0, st>>>(*L, sg, ws, nzx);
            if (int rc = launch_error(fn)) return rc;
        }
    }
    return FCN_OK;
}

extern "C" long long fcn_train_workspace_floats(const fcn_train_layer *L) {
    // enough for the split the launcher would like to use: SPLIT_CTAS CTAs' worth of partial tiles, at most K/32 slices
    if (L == nullptr || !shape_ok(*L)) return 0;
    return train_plan(*L, FWD_UNBOUNDED).partial;
}

extern "C" long long fcn_train_deterministic_workspace_floats(const fcn_train_layer *L) {
    if (L == nullptr || !shape_ok(*L)) return 0;
    return det_floats(*L);
}

extern "C" int fcn_train_forward(const fcn_train_layer *L, float *workspace, long long workspace_floats,
                                 fcn_stream_t stream) {
    return train_forward(__func__, L, workspace, workspace_floats, false, (cudaStream_t)stream);
}

extern "C" int fcn_train_forward_deterministic(const fcn_train_layer *L, float *workspace, long long workspace_floats,
                                               fcn_stream_t stream) {
    return train_forward(__func__, L, workspace, workspace_floats, true, (cudaStream_t)stream);
}

extern "C" int fcn_train_backward(const fcn_train_layer *L, int need_dx_mask, fcn_stream_t stream) {
    return train_backward(__func__, L, need_dx_mask, nullptr, 0, false, (cudaStream_t)stream);
}

extern "C" int fcn_train_backward_deterministic(const fcn_train_layer *L, int need_dx_mask, float *workspace,
                                                long long workspace_floats, fcn_stream_t stream) {
    return train_backward(__func__, L, need_dx_mask, workspace, workspace_floats, true, (cudaStream_t)stream);
}

extern "C" int fcn_train_pool(const fcn_train_pool_args *P, int backward, fcn_stream_t stream) {
    FCN_REQUIRE(P != nullptr, "NULL args");
    FCN_REQUIRE(P->B >= 1 && P->T >= 1 && P->K >= 1 && P->C >= 1 && P->V >= 0, "bad shape");
    FCN_REQUIRE(P->Y && P->cnt && P->argmax && P->sums && P->gamma && P->beta, "NULL pointer");
    dim3 grid(P->B * P->T, ceil_div(P->C + P->V, 128));
    if (!backward) {
        FCN_REQUIRE(P->feat && (P->V == 0 || P->one_hot), "NULL feature / one-hot pointer");
        train_pool_fwd_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(*P);
    } else {
        FCN_REQUIRE(P->dA && P->dfeat, "NULL gradient pointer");
        train_pool_bwd_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(*P);
    }
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

extern "C" int fcn_train_finalize(const fcn_train_layer *layers_dev, int n_layers, int update_running,
                                  fcn_stream_t stream) {
    FCN_REQUIRE(layers_dev != nullptr && n_layers >= 1, "bad layer table");
    train_finalize_kernel<<<n_layers, 128, 0, (cudaStream_t)stream>>>(layers_dev, n_layers, update_running);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

extern "C" int fcn_adam_step(float *param, const float *grad, float *exp_avg, float *exp_avg_sq, long long n, float lr,
                             float beta1, float beta2, float eps, float weight_decay, int step, float grad_scale,
                             fcn_stream_t stream) {
    FCN_REQUIRE(param && grad && exp_avg && exp_avg_sq && n >= 0 && step >= 1, "bad arguments");
    if (n == 0) return FCN_OK;
    const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
    const int threads = 256;
    train_adam_kernel<<<(unsigned)((n + threads - 1) / threads), threads, 0, (cudaStream_t)stream>>>(
        param, grad, exp_avg, exp_avg_sq, (size_t)n, lr, beta1, beta2, eps, weight_decay, bc1, bc2, grad_scale);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

extern "C" int fcn_sgd_step(float *param, const float *grad, float *momentum_buffer, long long n, float lr,
                            float momentum, float weight_decay, int first, float grad_scale, fcn_stream_t stream) {
    FCN_REQUIRE(param && grad, "NULL param / grad");
    FCN_REQUIRE(momentum == 0.f || momentum_buffer, "NULL momentum_buffer with momentum != 0");
    FCN_REQUIRE(n >= 0, "n < 0");
    if (n == 0) return FCN_OK;
    const int threads = 256;
    train_sgd_kernel<<<(unsigned)((n + threads - 1) / threads), threads, 0, (cudaStream_t)stream>>>(
        param, grad, momentum_buffer, (size_t)n, lr, momentum, weight_decay, first, grad_scale);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

// ------------------------------------------------------------------ rank-ordered fold of G gradient shards
// dst[i] = ((src[i] + src[ld+i]) + src[2ld+i]) + ... + src[(G-1)ld+i], every add __fadd_rn (no FMA contraction can
// touch it), so the sum has one order whatever the transport that gathered the G rows.  One thread per float4 of the
// body when src, ld and dst allow 16-byte access; the threads past the body take the n % 4 tail elements one each.
namespace fcn {

template <bool V4>
__global__ void __launch_bounds__(256) rank_fold_kernel(const float *__restrict__ src, long long ld, int G,
                                                        long long n, float *__restrict__ dst) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long j = i;
    if (V4) {
        const long long n4 = n >> 2;
        if (i < n4) {
            const float4 *s = reinterpret_cast<const float4 *>(src) + i;
            const long long ld4 = ld >> 2;
            float4 a = __ldg(s);
#pragma unroll 4
            for (int r = 1; r < G; ++r) {
                const float4 b = __ldg(s + r * ld4);
                a.x = __fadd_rn(a.x, b.x);
                a.y = __fadd_rn(a.y, b.y);
                a.z = __fadd_rn(a.z, b.z);
                a.w = __fadd_rn(a.w, b.w);
            }
            reinterpret_cast<float4 *>(dst)[i] = a;
            return;
        }
        j = 4 * n4 + (i - n4);
    }
    if (j >= n) return;
    float a = __ldg(src + j);
#pragma unroll 4
    for (int r = 1; r < G; ++r) a = __fadd_rn(a, __ldg(src + r * ld + j));
    dst[j] = a;
}

}  // namespace fcn

extern "C" int fcn_rank_fold(const float *src, long long ld, int G, long long n, float *dst, fcn_stream_t stream) {
    FCN_REQUIRE(src != nullptr && dst != nullptr, "NULL src / dst");
    FCN_REQUIRE(G >= 1, "G < 1");
    FCN_REQUIRE(n >= 0, "n < 0");
    FCN_REQUIRE(ld >= n, "ld < n");
    FCN_REQUIRE(G == 1 || ld <= (INT64_MAX / 4 - n) / (G - 1), "(G - 1) * ld + n overflows the address range");
    const uintptr_t s0 = (uintptr_t)src, s1 = s0 + 4 * (uintptr_t)((long long)(G - 1) * ld + n);
    const uintptr_t d0 = (uintptr_t)dst, d1 = d0 + 4 * (uintptr_t)n;
    FCN_REQUIRE(n == 0 || d1 <= s0 || s1 <= d0, "dst overlaps src");
    if (n == 0) return FCN_OK;
    const bool v4 = ((s0 | d0) & 15) == 0 && (ld & 3) == 0;
    const long long threads = v4 ? (n >> 2) + (n & 3) : n;
    const unsigned blocks = (unsigned)((threads + 255) / 256);
    if (v4)
        rank_fold_kernel<true><<<blocks, 256, 0, (cudaStream_t)stream>>>(src, ld, G, n, dst);
    else
        rank_fold_kernel<false><<<blocks, 256, 0, (cudaStream_t)stream>>>(src, ld, G, n, dst);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}
