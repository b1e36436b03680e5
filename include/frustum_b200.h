/*
 * frustum_b200.h — C ABI of libfrustum_b200.so (sm_90a).
 *
 * Drop-in boundary for the per-frustum hot path of Gorilla-Lab-SCUT/frustum-convnet:
 *   ops/query_depth_point  ->  models/det_base.PointNetFeat  ->  ConvFeatNet  ->  heads/decode.
 *
 * Conventions (SURVEY.md section 8(b)):
 *   - plain pointers + sizes only; every pointer is a DEVICE pointer unless the name says host;
 *   - the caller owns every buffer (the reference allocates outputs in Python and passes them
 *     in: ops/query_depth_point/query_depth_point.py:36-39); the library allocates nothing and
 *     keeps no state between calls except a thread-local error string;
 *   - `stream` is a cudaStream_t passed as void* (the reference launches on ATen's current
 *     stream: query_depth_point_cuda_kernel.cu:72); all calls are asynchronous;
 *   - return 0 on success, <0 on error (no C++ exception crosses the ABI; the reference raised
 *     through AT_ASSERTM / THCudaCheck: query_depth_point_cuda.cpp:5-10, ..._kernel.cu:85);
 *     fcn_last_error() returns the message of the last failing call on this thread.
 */
#ifndef FRUSTUM_B200_H_
#define FRUSTUM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FCN_OK 0
#define FCN_ERR_INVALID (-1)
#define FCN_ERR_CUDA (-2)

#define FCN_MAX_SCALES 8
#define FCN_MAX_SEGS 4

#if defined(__GNUC__)
#define FCN_API __attribute__((visibility("default")))
#else
#define FCN_API
#endif

typedef void *fcn_stream_t;

FCN_API int fcn_version(void);
FCN_API const char *fcn_last_error(void);

/* ------------------------------------------------------------------------------------------
 * (1) Grouping op.  Replaces query_depth_point_cuda.forward(b,n,m,dis_z,nsample,xyz1,xyz2,idx,
 *     pts_cnt) bound at ops/query_depth_point/query_depth_point_cuda.cpp:25-50 (kernel
 *     query_depth_point_cuda_kernel.cu:16-86).  Same argument order and meaning.
 *     idx: (b,m,nsample) int64, pts_cnt: (b,m) int32; both fully written (no pre-zero needed).
 *     _bn3  : xyz1 (b,n,3), xyz2 (b,m,3)   — the layout the reference kernel receives.
 *     _b3n  : xyz1 (b,3,n), xyz2 (b,3,m)   — the layout QueryDepthPoint.forward receives
 *             (query_depth_point.py:18-19); saves the two permute().contiguous() copies (:29-30).
 * ------------------------------------------------------------------------------------------ */
FCN_API int fcn_query_depth_point_bn3(int b, int n, int m, float dis_z, int nsample, const float *xyz1,
                              const float *xyz2, int64_t *idx, int32_t *pts_cnt,
                              fcn_stream_t stream);
FCN_API int fcn_query_depth_point_b3n(int b, int n, int m, float dis_z, int nsample, const float *xyz1,
                              const float *xyz2, int64_t *idx, int32_t *pts_cnt,
                              fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (2) Fused grouping -> row records (feeds the PointNet tile kernels; replaces
 *     QueryDepthPoint + torch.gather + "grouped_pc - new_pc", models/det_base.py:68-80,
 *     for all scales of PointNetFeat in ONE launch).
 *
 *     For every (frustum b, scale s) the T_s sections are scanned; section t contributes
 *     cnt = min(hits, K_s) rows (unique_rows=1) or exactly K_s rows with the reference's
 *     back-fill duplicates (unique_rows=0).  A row record is float4 {x-cx, y-cy, z-cz, bits(t)}
 *     (bits(t) = section index as int; sign bit set when the section is empty/masked).
 *     Rows of (b,s) are stored contiguously at rows[s] + b*row_cap[s]; record slots past them
 *     are not written.  Tiles of `tile_rows` rows are appended to tiles[s] (int4 {b, row0,
 *     nrows, 0}), the tiles of one frustum in consecutive slots; ntiles[s] counts all of them
 *     but only the first tile_cap[s] are stored.
 *     Side outputs: cnt[s] (B,T_s) int32; rows [0,T_s) of each frustum's block of feat[s]
 *     (B,feat_pitch[s],ld_feat[s]) fp32 position-major are zero-filled and their one-hot
 *     channels [c3[s], c3[s]+num_vec) written (det_base.py:145-157); rows [T_s, feat_pitch[s])
 *     are not written.
 *     idx_scratch[s] is caller-provided scratch of (B,T_s,K_s) int32, required on every path;
 *     its contents after the call are unspecified.
 *     `ntiles` (int32[FCN_MAX_SCALES]) is reset by the call itself, every entry of it.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    int num_scales, B, N, num_vec, tile_rows, unique_rows;
    const float *pc;                        /* (B,3,N) */
    const float *one_hot;                   /* (B,num_vec) or NULL */
    const float *centers[FCN_MAX_SCALES];   /* (B,3,T_s) */
    int T[FCN_MAX_SCALES], K[FCN_MAX_SCALES];
    float dis_z[FCN_MAX_SCALES];
    int c3[FCN_MAX_SCALES], ld_feat[FCN_MAX_SCALES];
    int row_cap[FCN_MAX_SCALES];            /* rows reserved per frustum (>= T_s*K_s) */
    int tile_cap[FCN_MAX_SCALES];           /* capacity of tiles[s] */
    void *rows[FCN_MAX_SCALES];             /* float4[B*row_cap] */
    int32_t *cnt[FCN_MAX_SCALES];           /* (B,T_s) */
    float *feat[FCN_MAX_SCALES];            /* (B,T_s,ld_feat) or NULL */
    void *tiles[FCN_MAX_SCALES];            /* int4[tile_cap] */
    int32_t *idx_scratch[FCN_MAX_SCALES];   /* (B,T_s,K_s) int32 scratch, contents unspecified after the call */
    int feat_pitch[FCN_MAX_SCALES];         /* rows per frustum of feat[s] (>= T_s; 0 means T_s) */
    int32_t *ntiles;                        /* int32[FCN_MAX_SCALES] */
    int force_scan;                         /* 1: section-scan kernel pair instead of the bit-matrix kernel (A/B) */
} fcn_group_args;
FCN_API int fcn_group_rows(const fcn_group_args *args, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (3) PointNet tile kernel: three folded (conv1x1 + BN + ReLU) layers on row tiles and the
 *     max over the rows of each section.  Replaces models/det_base.py:95-101 + torch.max(-1)
 *     (:134-143) for one scale.
 *     Weights are BN-folded and packed by the host side (see INTEGRATION.md):
 *       w1t (3,C1)  w2t (C1,C2)  w3t (C2,C3)  fp32 row-major [cin][cout];  b1,b2,b3 fp32.
 *     pooled   : out = feat (B,T,ld_feat) position-major, combined with atomic max (feat must be
 *                zero-initialised, which fcn_group_rows does).
 *     unpooled : out = (B,C3,T,K) channel-first un-pooled masked tensor — the return value of
 *                PointNetModule.forward (det_base.py:103); rows must come from unique_rows=0.
 *     precision: 0 = fp32 SIMT, 1 = TF32 tensor cores (wgmma) for the C1->C2->C3 layers,
 *                2 = same on 2-CTA clusters, weight stages multicast to both CTAs (C1 >= 128).
 *     Tiles: the rows of one section are contiguous within a tile (a section may continue in another tile);
 *     record slots past a tile's nrows are never read.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    int C1, C2, C3, T, K, ld_feat, row_cap, tile_rows, unpooled, precision, B;
    const void *rows;       /* float4 records of this scale */
    const void *tiles;      /* int4 tile table */
    const int32_t *ntiles;  /* device scalar */
    int max_tiles;          /* host upper bound used to size the grid */
    const float *w1t, *b1, *w2t, *b2, *w3t, *b3;
    const void *w2_tc, *w3_tc;  /* tensor-core packed images (precision=1), else NULL */
    float *out;
    long long *dbg_clocks;  /* optional (NULL): CTA 0 dumps pipeline timestamps (diagnostics) */
    int feat_pitch;         /* rows per frustum of the pooled feature map (>= T; 0 means T) */
} fcn_pointnet_args;
FCN_API int fcn_pointnet_tiles(const fcn_pointnet_args *args, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (4) 1-D conv / transposed conv / 1x1 conv + folded BN + optional ReLU as an implicit GEMM on
 *     position-major activations.  Replaces every Conv1d/DeConv1d block of ConvFeatNet
 *     (models/det_base.py:167-224, factories models/common.py:38-63), the torch.cat calls
 *     (multi-segment A operand) and the two heads (det_base.py:367-368).
 *       precision: 0 fp32 SIMT | 1,2 TF32 wgmma with cp.async gather (N tile 128|64) |
 *                  3,4 TF32 wgmma fully TMA-fed (N tile 128|64, needs `tmaps`)
 *       out[b, t*up + j, c_off + co] = act( sum_seg sum_c src[b, t*stride + tap, c] * W + bias )
 *     K is the concatenation of the segments, each padded to a multiple of 32 (zero weights); K_pad
 *     is that sum, optionally rounded up to a multiple of 64 (required by the tensor-core variants).
 *     The channel pad [C, ld) of a source is read (against those zero weights) and must hold finite values.
 *     wt: [K_pad][n_cols] fp32 (n_cols = up*Cout rounded up to 64), bias: [n_cols].
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    const float *src;
    int ld, C, T_src, tap, stride;
    int pitch;   /* rows per frustum of src (>= T_src; 0 means T_src).  Padded maps (pitch > T_src, pad rows
                    kept zero) let the GEMM run over the flattened (frustum, position) rows: the kernel
                    taps then read a zero pad row instead of the neighbouring frustum. */
} fcn_conv_seg;
typedef struct {
    int B, T_out, n_seg;
    fcn_conv_seg seg[FCN_MAX_SEGS];
    int K_pad, n_cols, Cout, up, relu, precision;
    const float *wt, *bias;
    const void *w_tc;
    float *out;
    int ld_out, T_store, c_off;
    int round_out;   /* 1: round outputs to TF32 (cvt.rna) because a tensor-core GEMM consumes them */
    long long *dbg_clocks; /* optional (NULL): CTA (0,0) dumps per-K-block pipeline timestamps, 8 per K block */
    const void *tmaps;     /* HOST pointer to n_seg 128-byte tensor maps (precision 3|4), see below */
    int P_m;               /* pitch of the GEMM row space: row r = b*P_m + t, valid iff t < T_out (0: T_out) */
    int P_store;           /* rows per frustum of `out` (>= T_store; 0 means T_store) */
} fcn_conv_args;
FCN_API int fcn_conv_gemm(const fcn_conv_args *args, fcn_stream_t stream);

/* TMA descriptor of a position-major activation map (B,T,ld) fp32 for the fully TMA-fed conv GEMM
 * (precision 3 = N tile 128, 4 = N tile 64): 3-D tensor (channel, position, frustum), box
 * 32 x 128 x 1 with 128-byte swizzle, position step t_stride (1, or 2 for the stride-2 convs).
 * The kernel addresses the GEMM rows as ONE flattened sequence, so encode the map with B = 1 and
 * T = (number of frustums) x pitch of the padded activation map.
 * Writes 128 bytes to HOST memory; pass an array of them (one per segment) in fcn_conv_args.tmaps. */
FCN_API int fcn_encode_activation_map(void *out_map_128B, const float *base, int B, int T, int ld,
                                      int t_stride);

/* ------------------------------------------------------------------------------------------
 * (5) Eval decode of the head logits.  Replaces models/det_base.py:376-411 and
 *     models/box_transform.py:5-12,28-41.
 *     logits: (B, pitch >= T, ld) rows = [cls0, cls1, center(3), heading scores(NH), heading res(NH),
 *     size scores(NS), size res(NS*3)];  center_ref: (B,3,T) channel-first;  mean_size (NS,3).
 * ------------------------------------------------------------------------------------------ */
FCN_API int fcn_decode_eval(int B, int T, int pitch, int ld, int num_heading_bin, int num_size, const float *logits,
                    const float *center_ref, const float *mean_size, float *cls_probs,
                    float *center, float *heading, float *size, float *heading_probs,
                    float *size_probs, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (5b) Persistent FCN kernel: every fcn_conv_gemm layer of ConvFeatNet + heads (4) and the eval decode (5) of
 *      one forward in ONE launch (models/det_base.py:196-224,367-411).  The host describes the network as
 *        layers : per layer the A segments (tensor-map index, 32-channel blocks, kernel tap, stride), the
 *                 packed TF32 weight image / bias, the output slice and the index of its completion counters;
 *        jobs   : one [128 rows x NT columns] output tile each, in TOPOLOGICAL order (a job depends only on jobs
 *                 with a smaller index), with the counters (first, count, target) it has to wait for;
 *        tmaps  : HOST array of n_maps (<= 48) 128-byte tensor maps - A-operand load maps
 *                 (fcn_encode_activation_map) and epilogue store maps (fcn_encode_store_map); copied into the
 *                 kernel parameters at launch, like the HOST layer table;
 *        sync   : DEVICE int32[4 + n_flags], zero-initialised ONCE by the caller; [0] job counter, [1] finished
 *                 CTAs, [2] epoch (forwards completed), [4..] per-(layer,row-tile) completion counters.  The
 *                 kernel resets [0],[1],[4..] itself at the end of every forward.  A finished tile of a
 *                 non-heads layer adds 1 to its row tile's counter, so a row tile of a layer with n_tiles_n column
 *                 tiles is complete at n_tiles_n.
 *      The bias of a non-heads layer is bulk-copied in NT-column slices and must be 16-byte aligned.
 *      Persistent CTAs fetch jobs with an atomic counter (deadlock-free under any co-residency, see fcn_mega.cu).
 *      The heads layer (is_heads) stores the logits row and decodes it in place into `n_out` output sets:
 *      outs[0] is the local 6-tuple block, outs[1..] are peer buffers (mapped NVLink peer memory) - the
 *      multi-GPU result exchange without a collective; flag_out[i] (may be NULL) receives the epoch number when
 *      the forward is complete (system-scope release).
 * ------------------------------------------------------------------------------------------ */
#define FCN_MAX_PEERS 8
#define FCN_MEGA_MAX_DEPS 4
typedef struct {
    float *cls_probs, *center, *heading, *size, *heading_probs, *size_probs;
} fcn_decode_out;
typedef struct {
    int map_idx, kblocks, tap, stride;
} fcn_mega_seg;
typedef struct {
    int n_seg;
    fcn_mega_seg seg[FCN_MAX_SEGS];
    int n_stage;                 /* weight-image stages per tile: K_pad / (32 * k_atoms) */
    int NT, n_tiles_n;           /* N tile (256 | 128 | 64) and their number */
    int relu, round_out, up, Cout;
    int P_m, T_out, n_rows;      /* GEMM row space: row r = b*P_m + t, valid iff t < T_out; n_rows = B*P_m */
    int ld_out, P_store, T_store, c_off;
    int is_heads, flag_base;
    int out_map;                 /* tensor map of the epilogue's TMA stores (fcn_encode_store_map); unused for heads */
    int k_atoms;                 /* 32-wide K atoms per weight-image stage: 2 (NT <= 128) or 1 (NT = 256); the kernel
                                    streams n_stage * k_atoms stages of one atom each */
    const void *w_tc;            /* packed stage images, N-tile major */
    const float *bias;
    float *out;
} fcn_mega_layer;
typedef struct {
    int first, count, target;
} fcn_mega_dep;
typedef struct {
    int layer, m_tile, n_tile, n_dep;
    fcn_mega_dep dep[FCN_MEGA_MAX_DEPS];
} fcn_mega_job;
typedef struct {
    int n_layers, n_jobs, n_flags, grid;   /* grid: persistent CTAs (0 = one per SM) */
    const fcn_mega_layer *layers;          /* HOST, n_layers (<= 24) records */
    const fcn_mega_job *jobs;              /* device */
    const void *tmaps;                     /* HOST, n_maps x 128 bytes */
    int32_t *sync;                         /* device */
    int n_maps, reserved0;
    int B, T, NH, NS;                      /* decode: frustums, positions (T2), heading bins, size clusters */
    const float *center_ref, *mean_size;
    int n_out, n_flag_out;
    fcn_decode_out outs[FCN_MAX_PEERS];
    int32_t *flag_out[FCN_MAX_PEERS];
    long long *dbg_clocks;                 /* optional (NULL): phase timeline, 32 clocks per job for the first 64
                                              jobs of every CTA (grid x 64 x 32 values; fcn_mega.cu) */
} fcn_mega_args;
FCN_API int fcn_mega_forward(const fcn_mega_args *args, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (5c) Multi-GPU plumbing for the result exchange by peer stores (one process per GPU): export a caller-owned
 *      device buffer as a CUDA-IPC handle (+ the byte offset of `dev_ptr` inside its allocation), map an
 *      exported buffer into this process for the current device, unmap it.  The mapped address (+ offset) is what
 *      fcn_mega_args.outs[1..] / flag_out[] take.  handle = 64 bytes of HOST memory.
 * ------------------------------------------------------------------------------------------ */
FCN_API int fcn_ipc_export(const void *dev_ptr, void *handle_64B, long long *offset_bytes);
FCN_API int fcn_ipc_open(const void *handle_64B, void **base_out);
FCN_API int fcn_ipc_close(void *base);

/* TMA descriptor for the epilogue stores of the persistent FCN kernel: a position-major map viewed as
 * (inner = up*ld floats, rows = flattened GEMM rows), box 32 x 32 with 128-byte swizzle.  For a transposed conv
 * with `up` taps the GEMM row r, tap j lands on output row r*up + j: one tensor row = `up` consecutive output
 * rows, the tap selects the inner offset j*ld.  Writes 128 bytes to HOST memory. */
FCN_API int fcn_encode_store_map(void *out_map_128B, const float *base, int rows, int inner);

/* ------------------------------------------------------------------------------------------
 * (7) Training step (config 5, cfgs/refine_car.yaml): PointNetDet in train() mode on hand-written kernels.
 *     Replaces the PyTorch/cuDNN autograd graph of models/det_base.py:62-224,367-368 (+ models/common.py:38-63
 *     BatchNorm in batch-statistics mode) and the optimizer step (train/train_net_det.py:121-128,322-323).
 *     All tensors are dense position-major fp32 [rows, channels]; rows = (frustum, position).  A layer is
 *         Y = act(X) * W (+bias)          act = the PRODUCER's BatchNorm (batch statistics) + ReLU, applied while
 *                                         the operand is loaded (no post-activation tensor exists)
 *     and its backward applies the BatchNorm/ReLU backward on the fly as well (see csrc/train.cu).
 *     Weights / gradients are addressed in the PARAMETER layout through strides:
 *         W[segment channel c, column n] = W + w_off + c*s_ci + (n % Cout)*s_co + (n / Cout)*s_j
 *     fcn_train_src: how a consumer sees a source tensor: position p of frustum b, channel c ->
 *         raw[(b*T + p/up)*ld + c0 + (p%up)*cup + c]   (up > 1: un-shuffled output of a transposed conv)
 *     `sums` (fp64 [2*Cstat]: Sum(y), Sum(y^2)) non-NULL = the source is a BN layer's raw output: apply
 *     gamma*(y-mean)*invstd+beta (channel (coff + c) % Cstat, `count` samples per channel) and ReLU if `relu`.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    const float *raw;
    float *grad;                 /* gradient w.r.t. the POST-activation values, same layout as raw (may be NULL) */
    const double *sums;
    const float *gamma, *beta;
    double count;
    int Cstat, coff, relu;
    int ld, T, up, cup, c0;
} fcn_train_src;
typedef struct {
    fcn_train_src src;
    int C, tap, stride, s_ci;
    long long w_off;
} fcn_train_seg;
typedef struct {
    int B, T_out, n_seg, N, Cout, up, s_co, s_j, has_bn, relu;
    fcn_train_seg seg[FCN_MAX_SEGS];
    const float *W;
    float *dW;
    const float *bias;           /* plain (no BN) layers only, else NULL */
    float *dbias;
    float *Y;                    /* raw output [B*T_out, N] */
    float *dA;                   /* gradient w.r.t. this layer's post-activation output [B*T_out, N] */
    double *sums;                /* [2*Cout] Sum(y), Sum(y^2): zeroed by the caller before the forward */
    double *dsums;               /* [2*Cout] Sum(dz), Sum(dz*xh): zeroed by the caller before the backward */
    const float *gamma, *beta;
    float *dgamma, *dbeta, *run_mean, *run_var;
} fcn_train_layer;
/* `workspace` (may be NULL): scratch for the K-split of skinny layers (partial sums, added in a fixed order);
 * fcn_train_workspace_floats(layer) = the size the launcher would like for this layer. */
FCN_API long long fcn_train_workspace_floats(const fcn_train_layer *layer);
FCN_API int fcn_train_forward(const fcn_train_layer *layer, float *workspace, long long workspace_floats,
                              fcn_stream_t stream);
/* backward of one layer: column reduction, dW (all segments), dX for the segments in need_dx_mask.
 * Every output of the training kernels except Y ACCUMULATES into what its buffer holds: dX (into src.grad, so a
 * source read by several segments or layers receives the sum of their gradients), dW, dbias, dgamma / dbeta,
 * `sums` and `dsums`.  The forward OVERWRITES Y. */
FCN_API int fcn_train_backward(const fcn_train_layer *layer, int need_dx_mask, fcn_stream_t stream);
/* Deterministic mode: the same layer forward / backward with bit-reproducible results.  No float atomics: partial
 * results go to `workspace` with plain stores and are added in a fixed order (BN statistics and Sum(dz), Sum(dz*xh)
 * as fp32 per-row-block column sums added in fp64; dW and dX as fp32 slices added in slice order, then added once to
 * the accumulating buffer).  Every split depends on the layer's shape only, never on the workspace offered or on the
 * device, so one build gives the same bits for the same inputs on every run, stream and graph replay, whatever the
 * workspace held before.  The accumulation contract of fcn_train_forward / fcn_train_backward holds.  The bits
 * differ from the default path's (another summation order).
 * fcn_train_deterministic_workspace_floats(layer): the floats both entries need, from the layer's shape and its
 * structure only: its sizes, taps and strides, the layout strides and offsets that decide between the plain and
 * the generic kernels, and whether `bias` is NULL (a BN layer with a bias cannot take the plain kernels, whose
 * split differs).  No pointer is dereferenced and no device is needed;
 * 0 for a NULL layer or a bad shape.  A NULL workspace or one with
 * fewer floats returns FCN_ERR_INVALID before anything is launched.  Calls on one stream may share one workspace. */
FCN_API long long fcn_train_deterministic_workspace_floats(const fcn_train_layer *layer);
FCN_API int fcn_train_forward_deterministic(const fcn_train_layer *layer, float *workspace, long long workspace_floats,
                                            fcn_stream_t stream);
FCN_API int fcn_train_backward_deterministic(const fcn_train_layer *layer, int need_dx_mask, float *workspace,
                                             long long workspace_floats, fcn_stream_t stream);
/* PointNet pooling: feat[(b,t), c] = (cnt > 0) * max_k relu(bn(Y[(b,t,k), c])), one-hot columns appended
 * (det_base.py:100-101,134-157); backward scatters dfeat to the arg-max rows of a zero-filled dA. */
typedef struct {
    int B, T, K, C, V, ld_feat;
    const float *Y;
    const int32_t *cnt;
    const double *sums;
    const float *gamma, *beta, *one_hot;
    float *feat;
    int32_t *argmax;
    const float *dfeat;
    float *dA;
} fcn_train_pool_args;
FCN_API int fcn_train_pool(const fcn_train_pool_args *args, int backward, fcn_stream_t stream);
/* end of step, one launch for all layers (DEVICE copy of the layer table): running statistics (momentum 0.1,
 * unbiased variance), dgamma / dbeta / dbias from the reduction buffers */
FCN_API int fcn_train_finalize(const fcn_train_layer *layers_dev, int n_layers, int update_running,
                               fcn_stream_t stream);
/* fused Adam over one flat bucket (torch.optim.Adam semantics incl. L2 weight decay); grad_scale multiplies
 * the gradient first (1/world after a sum all-reduce) */
FCN_API int fcn_adam_step(float *param, const float *grad, float *exp_avg, float *exp_avg_sq, long long n, float lr,
                          float beta1, float beta2, float eps, float weight_decay, int step, float grad_scale,
                          fcn_stream_t stream);
/* fused SGD over one flat bucket (torch.optim.SGD with momentum and L2 weight decay; no nesterov, dampening or
 * maximize), the operations and roundings of torch's single-tensor step: d = g*grad_scale (+ wd*p when wd != 0);
 * with momentum != 0, momentum_buffer = d when `first` (torch's first step with momentum), else
 * momentum_buffer*momentum + d, and d = momentum_buffer; then p += (-lr)*d.  The two "+ alpha*y" steps are single
 * FMAs, as torch's CUDA add(x, y, alpha=) computes them.  grad_scale multiplies the gradient first (1/world after a
 * sum all-reduce; exactly 1 on one rank).  n == 0 is a no-op.  momentum_buffer may be NULL when
 * momentum == 0 (then it is neither read nor written). */
FCN_API int fcn_sgd_step(float *param, const float *grad, float *momentum_buffer, long long n, float lr,
                         float momentum, float weight_decay, int first, float grad_scale, fcn_stream_t stream);
/* rank-ordered fold of G rows of n floats, row r at src + r*ld (the G ranks' shards of a gradient piece, as an
 * all-to-all leaves them): dst[i] = ((src[i] + src[ld+i]) + src[2ld+i]) + ... + src[(G-1)ld+i], a left fold in rank
 * order with every add rounded on its own (no FMA), so the sum does not depend on how the rows were gathered.
 * G == 1 is a copy.  One thread per float4 where src, dst and ld allow 16-byte access, per float otherwise; no
 * atomics.  NULL pointers, G < 1, n < 0, ld < n, or dst overlapping [src, src + (G-1)*ld + n) return
 * FCN_ERR_INVALID before anything is launched; n == 0 is a no-op. */
FCN_API int fcn_rank_fold(const float *src, long long ld, int G, long long n, float *dst, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (7b) Fused detection losses + gradient w.r.t. the head logits (row 8(f)-2, train half): everything of
 *      models/det_base.py:414-503 after the heads - foreground selection, focal loss (models/common.py:217-232),
 *      Huber / cross-entropy / corner losses (models/model_util.py:9-72, models/box_transform.py:5-65), accuracies
 *      and the rotated-IoU metrics - and its autograd backward, in three tiny launches.
 *      cls (B*T2, 2), reg (B*T2, 3 + 2*NH + 4*NS) rows in (frustum, position) order; labels as the reference's
 *      data dict holds them (cls_label int64 (B,T2) in {-1,0,1}, size_class int64 (B), box3d_* fp32).
 *      out[0..7] = total, cls, center, head_cls, head_res, size_cls, size_res, corners; out[8..13] = cls_acc,
 *      head_acc, size_acc, IoU_2D, IoU_3D, IoU_>=thresh; out[14..15] = #foreground, #non-ignored rows.
 *      out[0] and out[8..10] follow the reference's float32 roundings: the total is det_base.py:468-474 in Python's
 *      evaluation order with every product and sum rounded on its own, and each accuracy is the float32 count times
 *      float32(1.0 / n), as get_accuracy (utils/utils.py:28-48) forms it.  fcn_val_batch forms its values the same way.
 *      scratch: 16 floats.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    int B, T2, NH, NS, with_iou, reserved0;
    const float *cls, *reg, *center_ref2 /* (B,3,T2) */;
    const long long *cls_label, *size_class;
    const float *box3d_center, *box3d_heading, *box3d_size, *mean_size /* (NS,3) */;
    float w_box, w_head_reg, w_size_reg, w_corner, iou_thresh, reserved1;
    float *dcls, *dreg, *out /* 16 floats */, *scratch /* 16 floats */;
} fcn_loss_args;
FCN_API int fcn_det_loss(const fcn_loss_args *args, fcn_stream_t stream);
/* Deterministic variant: the same outputs, with the 16 floats of `out` bit-reproducible (per-CTA sums added in CTA
 * order instead of float atomics); dcls / dreg are bit-identical to fcn_det_loss's.  `scratch` holds
 * fcn_det_loss_deterministic_scratch_floats(B*T2) floats (0 when rows is outside [1, 2^24]: beyond 2^24 rows the
 * float row counts would no longer be exact). */
FCN_API long long fcn_det_loss_deterministic_scratch_floats(long long rows);
FCN_API int fcn_det_loss_deterministic(const fcn_loss_args *args, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (8) Inference post-processing ("next" row 8(f)-4): batched rotated 3-D NMS on the device.  Replaces
 *     `cube_nms` = rotate_nms_3d_cc (ops/pybind11/rbbox_iou.py:294-311) -> rotate_non_max_suppression_3d_cpu
 *     (ops/pybind11/nms_cpu.h:148-240), called per image and class from train/test_net_det.py:126-152.
 *     dets: (total, 8) fp32 rows [cx, cy, cz, l, w, h, ry, score]; segment s = rows
 *     [seg_offsets[s], seg_offsets[s+1]) (one image x class list of at most fcn_rotate_nms_3d_max_dets() rows: only
 *     that many are considered, so callers split or refuse longer lists; nms.py refuses them); keep:
 *     (num_segments, keep_stride) int32 GLOBAL row indices in descending-score order (NaN scores first, equal
 *     scores by the larger index first), keep_count[s] <= top_k of them are valid.  A box is suppressed by a kept,
 *     higher-scored box when their axis-aligned bounding cubes overlap and the rotated 3-D IoU is >= thresh.
 * ------------------------------------------------------------------------------------------ */
FCN_API int fcn_rotate_nms_3d(int num_segments, const float *dets, const int32_t *seg_offsets, float thresh, int top_k,
                              int32_t *keep, int32_t *keep_count, int keep_stride, fcn_stream_t stream);
FCN_API int fcn_rotate_nms_3d_max_dets(void);

/* ------------------------------------------------------------------------------------------
 * (9) Device-side input builder ("next" row 8(f)-3): ProviderDataset.__getitem__ of datasets/provider_sample.py
 *     (:133-203 resample + centre-view rotation, :291-327 generate_ref, datasets/data_utils.py:7-21,73-93) for a
 *     whole batch in one launch, from raw frustum points that stay resident in HBM.  `choice` (B,N) int32 = the
 *     caller's np.random.choice draw (indices into each frustum's own points).  float64 arithmetic with the
 *     reference's float32 casts.  Outputs have the layouts the model consumes: point_cloud (B,3,N),
 *     centers[s] (B,3,T_s), one_hot (B,num_classes) (optional), rot_angle (B) (optional).
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    int B, N, num_scales, num_classes;
    int T[FCN_MAX_SCALES];
    double stride[FCN_MAX_SCALES];
    const float *points;          /* (sum n_b, 3) raw frustum points, rect camera coordinates */
    const int32_t *point_offsets; /* (B+1) */
    const int32_t *choice;        /* (B, N) */
    const double *frustum_angle;  /* (B) */
    const double *box2d;          /* (B, 4) x1, y1, x2, y2 */
    const double *P;              /* (B, 12) calib P2, row-major 3x4 */
    const int32_t *cls_index;     /* (B) or NULL */
    float *point_cloud;
    float *centers[FCN_MAX_SCALES];
    float *one_hot;               /* or NULL */
    float *rot_angle;             /* or NULL */
} fcn_input_args;
FCN_API int fcn_build_inputs(const fcn_input_args *args, fcn_stream_t stream);

/* Layout helpers for the channel-first module APIs: (B,C,T) <-> (B,pitch >= T,ld) position-major. */
FCN_API int fcn_bct_to_btc(int B, int C, int T, int pitch, int ld, const float *src, float *dst,
                           fcn_stream_t stream);
FCN_API int fcn_btc_to_bct(int B, int C, int T, int pitch, int ld, const float *src, float *dst,
                           fcn_stream_t stream);

/* Self-test of the wgmma/bulk-copy building blocks: D (128,N) = A (128,K) * W^T with W given
 * as the pre-swizzled stage image of the host packer (engine.pack_sw128).  N in {64,128,256},
 * K multiple of 32 that fits shared memory: K <= 256 (N = 64), 224 (N = 128), 128 (N = 256).
 * Used by tests/ to pin the descriptor encodings on real hardware. */
FCN_API int fcn_selftest_umma(int N, int K, const float *A, const void *w_img, float *D,
                              fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (6) Train-branch metric ("next" row 8(f)-1): pairwise rotated-box IoU on the device.  Replaces the CPU
 *     Boost.Geometry call rbbox_iou_3d_pair (ops/pybind11/box_ops.h:173-260) and the device->host copy of
 *     the boxes in front of it (models/det_base.py:494-495).
 *     corners, qcorners: (M, 8, 3) fp32 box corners in the order of get_box3d_corners_helper
 *     (models/model_util.py:48-72), 16-byte aligned;  iou: (M, 2) = [BEV IoU, 3-D IoU] per pair, zeros when
 *     the bird's-eye-view polygons do not overlap (box_ops.h:199,226);  stats (optional, may be NULL): 3 floats
 *     = mean BEV IoU, mean 3-D IoU, fraction of pairs with 3-D IoU >= iou_thresh (det_base.py:497-500),
 *     reduced in a fixed order (deterministic).  M == 0 writes zeros to stats.
 * ------------------------------------------------------------------------------------------ */
FCN_API int fcn_rbbox_iou_3d_pair(int M, const float *corners, const float *qcorners, float *iou,
                                  float iou_thresh, float *stats, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (10) Per-image 3-D detections on the device.  Replaces the host loop of train/test_net_det.py:243-293
 *      (test_net_det_sunrgbd.py:197-252) and write_detection_results_nms (:126-152 / :120-145): foreground
 *      selection, from_prediction_to_label_format, the image x class grouping and rotated 3-D NMS of lists of
 *      any length.
 *
 *      fcn_det_candidates (once per batch, no host sync, capturable): one CTA per frustum b selects its
 *      foreground positions t (method 0 'nms': KITTI p0 < p1, SUN-RGBD p1 > 0.5, else the first argmax of p1;
 *      method 1 'top': the first argmax), scores them (KITTI p1 + rgb_prob, SUN-RGBD rgb_prob + max size_prob),
 *      decodes them in fp32 (ry = heading + rot_angle; centre rotated by -rot_angle about y, + ref_center,
 *      KITTI: ty += h/2), drops boxes with h, w or l < 0.01 and appends one record per row.  Rows are reserved
 *      with one atomicAdd on *counter per frustum; rows at or past `capacity` are counted but not written.
 *      seg_of_frustum[first + b] is the dense image x class id of frustum b.  rgb_prob (B) and ref_center
 *      (B,3) may be NULL (1 and 0).  Outputs are contiguous: cls_probs (B,T2,2), center (B,T2,3),
 *      heading (B,T2), size (B,T2,3) = (l, w, h), size_probs (B,T2,NS).
 *
 *      Finalize (once per pass, two calls around one host read of `info`):
 *        fcn_det_prepare : orders the records by (segment, frustum, t) - the reference's list order whichever
 *                          call or stream appended them - and, for 'nms', ranks every segment by descending
 *                          score (ties: larger list index first); writes seg_offsets (S+1) and
 *                          info = {rows counted, mask words needed, pair tiles, 0} (int64).
 *        fcn_det_select  : needs n_counted = info[0] <= capacity (else an error naming the capacity needed) and
 *                          a `mask` of >= info[1] words (no initialisation needed).  'nms': suppression bits of all
 *                          pairs of every segment (bounding cubes overlap, then rotated 3-D IoU >= thresh), tiled
 *                          32 x 32 over the whole grid; greedy scan per segment; keep[:top_k].  'top': every row.
 *                          rows (capacity, 12): kept row k of segment s at seg_offsets[s] + k, k < keep_count[s],
 *                          KITTI [x1,y1,x2,y2, tx,ty,tz, h,w,l, ry, score], SUN-RGBD [.., tx,ty,tz, l,w,h, ry, score],
 *                          box2d (num_frustums, 4) gives the first four columns.
 *      fcn_det_workspace_bytes = the workspace both finalize calls share (needs the device; -1 on error).
 * ------------------------------------------------------------------------------------------ */
#define FCN_DET_KITTI 0
#define FCN_DET_SUNRGBD 1
#define FCN_DET_NMS 0
#define FCN_DET_TOP 1
typedef struct {
    int32_t seg, frustum, t, reserved;
    float box[8];                  /* tx, ty, tz, l, w, h, ry, score: the NMS box and the label-format values */
} fcn_det_record;
typedef struct {
    int B, T2, NS, dataset, method, first, num_frustums, capacity;
    const float *cls_probs, *center, *heading, *size, *size_probs;
    const float *rot_angle, *rgb_prob, *ref_center;
    const int32_t *seg_of_frustum; /* (num_frustums) */
    int32_t *counter;              /* device scalar, zeroed by the caller before the pass */
    fcn_det_record *records;       /* (capacity) */
} fcn_det_candidate_args;
FCN_API int fcn_det_candidates(const fcn_det_candidate_args *args, fcn_stream_t stream);
typedef struct {
    int num_segments, num_frustums, capacity, method, dataset, top_k;
    float thresh;
    int n_counted;                 /* fcn_det_select: info[0] as read by the host */
    const int32_t *counter;
    const fcn_det_record *records;
    const float *box2d;            /* (num_frustums, 4) */
    void *workspace;
    long long workspace_bytes;
    long long *info;               /* device int64[4] */
    int32_t *seg_offsets;          /* (num_segments + 1) */
    int32_t *keep_count;           /* (num_segments) */
    float *rows;                   /* (capacity, 12) */
    uint32_t *mask;                /* fcn_det_select, method 'nms': >= info[1] words (may be NULL when info[1] == 0) */
    long long mask_words;
} fcn_det_finalize_args;
FCN_API long long fcn_det_workspace_bytes(int capacity, int num_segments);
FCN_API int fcn_det_prepare(const fcn_det_finalize_args *args, fcn_stream_t stream);
FCN_API int fcn_det_select(const fcn_det_finalize_args *args, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (11) Labelled training batches on the device: ProviderDataset.__getitem__ + collate for a whole batch in one
 *      launch (one CTA per item, no host sync, no allocation, capturable), from a dataset resident in HBM.
 *      cfg.DATA.RTC = True and WITH_EXTRA_FEAT = False only (every reference cfg); anything else is rejected.
 *        FCN_TRAIN_DET, labels = 1     datasets/provider_sample.py:133-270 (train branch), generate_labels :272-289,
 *                                      generate_ref :291-327, default_collate
 *        FCN_TRAIN_REFINE, labels = 1  datasets/provider_sample_refine.py:174-316 (train branch), generate_labels
 *                                      :318-334, generate_ref :336-385, collate_fn :388-419
 *        FCN_TRAIN_REFINE, labels = 0  the same file's from_rgb_detection branch :228-248 (no labels, no augmentation)
 *        FCN_TRAIN_SUNRGBD, labels = 1 datasets/provider_sample_sunrgbd.py:116-263 (train branch; with random_flip =
 *                                      random_shift = 0 the val split), generate_labels :265-280, generate_ref :283-326,
 *                                      default_collate; exactly 5 scales (the reference unpacks s1..s5)
 *        FCN_TRAIN_SUNRGBD, labels = 0 the same file's from_rgb_detection branch :165-186 (no labels, no augmentation)
 *      Per frustum the host stores one fcn_train_frustum of float64 values computed ONCE with the reference's own
 *      numpy expressions (exact by construction); per step only index (B), choice (B,N), flip_u (B), shift_n (B)
 *      cross PCIe (the caller's np.random draws, :164-166,227,241 / :207,270,284).  The kernel does the rest in
 *      float64 with every product and sum rounded separately, casting where numpy casts:
 *        point_cloud (B,3,N)   points[choice] rotated to the centre view (det: rot = pi/2 + frustum_angle, :157,354-362;
 *                              refine: minus the predicted centre, rotated by the predicted angle, :149-154,199), cast
 *                              to the dataset's dtype (points_f64 = 0: float32), x negated when flip_u > 0.5
 *                              (:227-235 / :270-278), z += shift (:237-244 / :280-286), then float32;
 *        centers[s] (B,3,P_s)  det: project_image_to_rect of the 2-D box centre at arange(0, max_depth, s) + s/2,
 *                              rotated; sunrgbd: project_image_to_upright_camera (:28-57) of the host's box-2D
 *                              centre (cx, cy) at the same depths - x = ((cx - K[0,2]) z) / K[0,0], y likewise with
 *                              K[1,2], K[1,1]; (x, z, -y); Rtilt @ that; (X, -Z, Y) - then rotated; refine: the
 *                              predicted box's line from its front to its back face mean at
 *                              arange(z_start, ., s) + s/2 (arange element i = z_start + i * z_step[s]); x negated by
 *                              the flip.  P_s = max over the batch of T[s] of the items (collate_fn :388-419 pads
 *                              with mode='edge': columns >= T[s] of an item repeat its last column);
 *        cls_label (B,P_2)     int64 on the float64 ref2: -1 inside the full box (det 1.0x, refine 0.6x the GT size),
 *                              1 inside the half box (det and sunrgbd 0.5x, refine 0.3x), 1 at the first argmin of
 *                              the distance to the GT centre when no ref is inside the half box; edge padded like the
 *                              refs.  The inside test is the half-space test in the box frame (the reference uses a Delaunay
 *                              triangulation of the 8 corners, data_utils.py:24-34: they differ within ~1e-15 m of a face);
 *        box3d_center (B,3), box3d_heading (B,1), box3d_size (B,3) float32, size_class (B,1) int64: the GT box in the
 *                              frame of the inputs, flipped (heading = pi - heading) and shifted like the points;
 *        seg_label (B,N)       int64 (det only), rot_angle (B,1), one_hot (B,num_classes) (NULL: none), ref_center
 *                              (B,3) (refine), rgb_prob (B,1) (labels = 0).  seg_label: det, and sunrgbd with labels.
 *      Shift: det and sunrgbd clip(n * dist * 0.2, +-0.5 dist), then clip(shift + c_z, 0, max_depth) - c_z; refine
 *      clip(n * dist * 0.1, +-2 stride[0]); dist = sqrt(l^2 + w^2) of the GT size.  sunrgbd then adds the height shift
 *      h = height_u * 0.4 - 0.2 (np.random.random(), :231-233, drawn after randn()) to the GT centre's y in float64 and
 *      to the points' y in float32 (numpy adds a Python float to a float32 array in float32).  sunrgbd's np.dot
 *      products (Rtilt @ and the centre-view rotation) follow OpenBLAS's dgemm order: the first product rounded, then
 *      one FMA per further term (its refs' centre-view x cancels to ~0, where the order shows).
 * ------------------------------------------------------------------------------------------ */
#define FCN_TRAIN_DET 0
#define FCN_TRAIN_REFINE 1
#define FCN_TRAIN_SUNRGBD 2
typedef struct {
    double rot, cs, sn;            /* rot_angle output and np.cos / np.sin of the centre-view rotation angle */
    double box2d[4], P[12];        /* det: 2-D box x1, y1, x2, y2 and calib P2 (row-major 3x4) */
    double ref_center[3];          /* refine: predicted box centre (pred_box3d[0] + pred_box3d[6]) / 2 */
    double line0[3], line_delta[3];/* refine: front face mean of the centre-view predicted box, back mean - front mean */
    double z_start;                /* refine: min z of the centre-view predicted box (the arange start) */
    double z_step[FCN_MAX_SCALES]; /* refine: (z_start + s) - z_start, numpy's arange increment */
    double center[3], heading;     /* GT centre and heading in the frame of the inputs (before flip / shift) */
    double size[3], dist;          /* GT size (l, w, h) and sqrt(l^2 + w^2) */
    double rgb_prob;               /* refine, labels = 0 */
    int32_t T[FCN_MAX_SCALES];     /* sections per scale (refine: len(np.arange(z_start, z_end, s))) */
    int32_t cls_index, reserved;   /* size class = one-hot index */
    double cx, cy;                 /* sunrgbd: (box[0] + box[2]) / 2., (box[1] + box[3]) / 2. in box2d's own dtype */
    double K[9], Rtilt[9];         /* sunrgbd: calib K and Rtilt (row-major 3x3) */
} fcn_train_frustum;
typedef struct {
    int kind, labels, rtc, extra_feat, random_flip, random_shift;
    int B, N, num_scales, num_classes, num_frustums, points_f64;
    double stride[FCN_MAX_SCALES];
    double max_depth;
    const void *points;                  /* (sum n, 3) float32, or float64 when points_f64 */
    const long long *point_offsets;      /* (num_frustums + 1) */
    const int32_t *seg;                  /* (sum n) det seg labels (label_list[i].astype(int64)), else NULL */
    const fcn_train_frustum *frustums;   /* (num_frustums) */
    const int32_t *index;                /* (B) dataset indices, repeats allowed */
    const int32_t *choice;               /* (B, N) indices into each item's own points */
    const double *flip_u, *shift_n;      /* (B) np.random.random() / np.random.randn() (read when enabled) */
    float *point_cloud;
    float *centers[FCN_MAX_SCALES];      /* (B, 3, P_s) contiguous, capacity B * 3 * max T[s] */
    long long *cls_label;                /* (B, P_2) */
    long long *seg_label;                /* (B, N) det */
    float *box3d_center, *box3d_heading, *box3d_size;
    long long *size_class;
    float *rot_angle, *one_hot, *ref_center, *rgb_prob;
    const double *height_u;              /* (B) sunrgbd: np.random.random() after randn() (read when shifting) */
} fcn_train_input_args;
FCN_API int fcn_build_train_inputs(const fcn_train_input_args *args, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (12) Validation pass on the device: the eval-mode losses and metrics of models/det_base.py:414-525 for every
 *      batch of an epoch, and their AverageMeter averages (utils/utils.py:51-67, utils/training_states.py).
 *
 *      fcn_val_batch (once per batch, after the eval forward; no host sync, no allocation, capturable): two
 *      launches.  Reads the head logits where the forward left them: logits (B, logit_pitch, ld_logit), row
 *      [cls0, cls1, centre 3, heading scores NH, heading residuals NH, size scores NS, size residuals 3*NS, ...];
 *      center_ref2 (B,3,T2); cls_label (B,T2) int64; size_class (B) int64; box3d_center (B,3), box3d_heading (B),
 *      box3d_size (B,3) fp32; mean_size (NS,3).  Computes the 8 losses and 6 metrics with the reference's
 *      denominators (focal loss / (nfg + 1e-14), cls_acc over label != -1, the rest over label == 1; IoU from the
 *      predicted classes; with_iou = 0 gives NaN IoU values).  Each CTA of the first launch writes its sums to
 *      its own slot of `partials` (fcn_val_partials_floats(B, T2) floats); the second sums the slots in CTA
 *      order, so results are bit-identical across runs, streams and graph replays (no float atomics).  It then
 *      appends one row to `table` (capacity, FCN_VAL_ROW) at row index state[0]++:
 *        [0..7]  total, cls, center, head_cls, head_res, size_cls, size_res, corners  (det_base.py:505-514)
 *        [8..13] cls_acc, head_acc, size_acc, IoU_2D, IoU_3D, IoU_>=thresh          (:516-523)
 *        [14] B, [15] nfg, [16] nkeep, [17] 0.
 *      state (device int32[4], zeroed by the caller at the start of an epoch): rows appended, status bits,
 *      index of the first batch without a foreground row (the reference's `assert fg_idx.numel() != 0`), 0.
 *      Rows at or past `capacity` are counted but not written (FCN_VAL_OVERFLOW).
 *
 *      fcn_val_finalize (once per epoch): one thread per value replays sum += (double)val * B, count += B with
 *      count starting at 1e-14, in row order, and writes avg = sum / count with the row count and status.
 *
 *      fcn_train_states_append (once per training step; no host sync, no allocation, capturable): one launch that
 *      appends a training step's losses and metrics to a table of the same layout, so the epoch's averages come
 *      from the same fcn_val_finalize.  `loss` is fcn_det_loss's `out` block (16 floats: the 14 values, #foreground,
 *      #non-ignored rows), B the step's batch size; the row is [14 values, B, nfg, nkeep, 0] at state[0]++, with
 *      state's status bits set as fcn_val_batch sets them.  capacity >= 1.
 * ------------------------------------------------------------------------------------------ */
#define FCN_VAL_VALUES 14
#define FCN_VAL_ROW 18
#define FCN_VAL_NO_FG 1
#define FCN_VAL_OVERFLOW 2
typedef struct {
    int B, T2, NH, NS, with_iou, capacity;
    int logit_pitch, ld_logit;
    const float *logits;
    const float *center_ref2;
    const long long *cls_label, *size_class;
    const float *box3d_center, *box3d_heading, *box3d_size, *mean_size;
    float w_box, w_head_reg, w_size_reg, w_corner, iou_thresh, reserved;
    float *partials;
    int32_t *state;
    float *table;
} fcn_val_batch_args;
typedef struct {
    double avg[FCN_VAL_VALUES], sum[FCN_VAL_VALUES], count;
    int32_t rows, added, status, first_no_fg;   /* rows in the table, rows appended (the capacity needed) */
} fcn_val_result;
FCN_API long long fcn_val_partials_floats(int B, int T2);
FCN_API int fcn_val_batch(const fcn_val_batch_args *args, fcn_stream_t stream);
FCN_API int fcn_val_finalize(const float *table, int capacity, const int32_t *state, fcn_val_result *result,
                             fcn_stream_t stream);
FCN_API int fcn_train_states_append(const float *loss, int B, float *table, int capacity, int32_t *state,
                                    fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (13) KITTI object evaluation on the device: the offline evaluator train/kitti_eval/evaluate_object_3d_offline.cpp
 *      (:56-916) with its semantics unchanged - image 2-D AP with AOS, ground-plane (bird's-eye-view) AP and 3-D AP
 *      for car, pedestrian and cyclist at the easy, moderate and hard levels, in float64 like the reference.
 *
 *      Records are float64 rows, one image after the other; image i owns rows [offsets[i], offsets[i+1]):
 *        gt  (num_gt, FCN_KITTI_GT_COLS)   [code, truncation, occlusion, alpha, x1, y1, x2, y2, h, w, l, t1, t2, t3, ry]
 *                                          (a label_2 line, loadGroundtruth :180-204, with the type as its code)
 *        det (num_det, FCN_KITTI_DET_COLS) [code, alpha, x1, y1, x2, y2, h, w, l, t1, t2, t3, ry, score]
 *                                          (a result line, loadDetections :133-178, without the two unused fields)
 *      Type codes FCN_KITTI_*: type names match case-insensitively; every other type is FCN_KITTI_OTHER.
 *      gt_offsets / det_offsets are DEVICE int32 arrays of num_images + 1 entries; host_gt_offsets /
 *      host_det_offsets are HOST copies of the same values (validated on the host and used for the buffer sizes:
 *      they must start at 0, never decrease and end at num_gt / num_det).
 *
 *      Three calls in order on one stream, sharing the caller's workspace (fcn_kitti_eval_workspace_bytes: reads
 *      neither workspace nor result, needs the device, -1 on invalid arguments), no host sync, no allocation:
 *        fcn_kitti_eval_overlaps   : run-level flags, and every (detection, ground truth) pair's overlap once per
 *                                    metric (criterion 0 against DontCare);
 *        fcn_kitti_eval_thresholds : per evaluation the TP scores, sorted, and the recall-step thresholds;
 *        fcn_kitti_eval_statistics : TP / FP / FN and AOS per threshold, then `result` (DEVICE).
 *      Results are bit-identical from run to run.  A class without a detection that enables a metric has
 *      evaluated[metric][class] = 0 and is not part of the output (its vectors are meaningless).
 * ------------------------------------------------------------------------------------------ */
#define FCN_KITTI_GT_COLS 15
#define FCN_KITTI_DET_COLS 14
#define FCN_KITTI_PTS 41
#define FCN_KITTI_CAR 0
#define FCN_KITTI_PEDESTRIAN 1
#define FCN_KITTI_CYCLIST 2
#define FCN_KITTI_VAN 3
#define FCN_KITTI_PERSON_SITTING 4
#define FCN_KITTI_DONTCARE 5
#define FCN_KITTI_OTHER 6
typedef struct {
    int num_images, num_gt, num_det, reserved0;
    const double *gt, *det;
    const int32_t *gt_offsets, *det_offsets;           /* DEVICE (num_images + 1) */
    const int32_t *host_gt_offsets, *host_det_offsets; /* HOST copies */
    void *workspace;
    long long workspace_bytes;
    struct fcn_kitti_eval_result_ *result;             /* DEVICE */
} fcn_kitti_eval_args;
typedef struct fcn_kitti_eval_result_ {
    double precision[3][3][3][FCN_KITTI_PTS];  /* [metric image|ground|3d][class][difficulty][recall step] */
    double aos[3][3][FCN_KITTI_PTS];           /* [class][difficulty][step]: image metric, when compute_aos */
    float ap[3][3][3];                         /* the printed AP: sum of steps 0, 4, ..., 40 in float32, / 11 * 100 */
    float ap_aos[3][3];
    int32_t n_thresholds[3][3][3];
    int32_t n_gt[3][3][3];                     /* recall denominators */
    int32_t evaluated[3][3];                   /* [metric][class] */
    int32_t compute_aos;                       /* no detection has alpha == -10 */
    int32_t reserved;
} fcn_kitti_eval_result;
FCN_API long long fcn_kitti_eval_workspace_bytes(const fcn_kitti_eval_args *args);
FCN_API int fcn_kitti_eval_overlaps(const fcn_kitti_eval_args *args, fcn_stream_t stream);
FCN_API int fcn_kitti_eval_thresholds(const fcn_kitti_eval_args *args, fcn_stream_t stream);
FCN_API int fcn_kitti_eval_statistics(const fcn_kitti_eval_args *args, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (14) SUN-RGBD 3-D detection evaluation on the device: eval_det / eval_det_cls of the reference
 *      (train/sunrgbd_eval/eval_det.py:41-231, use_07_metric = False) - per class the precision / recall curve and
 *      the VOC average precision, with the 3-D IoU of rbbox_iou_3d_pair<double> in float64.
 *
 *      Boxes are float64 corner sets (8, 3) in the reference's corner order; the bird's-eye-view ring is the (x, z) of
 *      corners 6, 7, 4, 5, the heights are the y of corners 0 and 4 (ops/pybind11/box_ops.h:173-260).  A ring that is
 *      not clockwise-positive scores 0 (as in csrc/box_iou.cuh).
 *        ground truth: class c owns rows [gt_class_offsets[c], gt_class_offsets[c+1]); within a class the rows are
 *                      grouped into segments, one per image: segment s owns rows [gt_segment_offsets[s], [s+1]), in
 *                      the reference's per-image order (the first maximum wins), and never crosses a class boundary.
 *        detections:   class c owns rows [det_class_offsets[c], [c+1]) in gather order; det_segments[d] is the
 *                      ground-truth segment of the detection's (class, image), or -1 when that image has no ground
 *                      truth of the class (the detection is a false positive).
 *      Per class: detections sorted by score, descending, STABLE (the earlier row wins a tie; -0.0 equals 0.0); the
 *      overlap maximum over the segment's rows in order with strict '>' (a NaN never wins); a hit needs ovmax >
 *      ovthresh strictly and is a TP when no higher-ranked detection claimed the same ground truth, otherwise an FP
 *      (no fall-back to another ground truth).  rec = tp / npos and prec = tp / max(tp + fp, DBL_EPSILON) are
 *      bit-identical to numpy's.  ap sums (delta recall) * (precision envelope) where the recall changes, in a fixed
 *      order (each of 512 threads sums its positions, one per 512-position chunk from the last chunk back, then
 *      cub::BlockReduce's fixed tree): within a few ulps of numpy's pairwise sum.  A class without a detection has
 *      nd = 0 and ap = 0.
 *
 *      gt_*_offsets / det_class_offsets are DEVICE int32 arrays; host_* are HOST copies of the same values (validated
 *      on the host: start at 0, never decrease, end at num_gt / num_det, class boundaries are segment boundaries).
 *      Two calls in order on one stream, sharing the caller's workspace (fcn_sunrgbd_eval_workspace_bytes: reads
 *      neither workspace nor outputs, needs the device, -1 on invalid arguments), no host sync, no allocation:
 *        fcn_sunrgbd_eval_match  : overlap maximum per detection, the per-class stable sort, the first claim of
 *                                  every ground truth;
 *        fcn_sunrgbd_eval_curves : rec / prec (DEVICE, num_det each, class c at [det_class_offsets[c], ...), in
 *                                  score order) and result[c] (DEVICE, num_classes entries).
 *      A det_segments entry outside [-1, num_gt_segments) or whose segment is not of the detection's class sets
 *      result[c].status to FCN_SUNRGBD_BAD_SEGMENT (the detection counts as an FP).  Results are bit-identical from run
 *      to run.
 * ------------------------------------------------------------------------------------------ */
#define FCN_SUNRGBD_MAX_CLASSES 1024
#define FCN_SUNRGBD_BAD_SEGMENT 1
typedef struct {
    int num_classes, num_gt, num_gt_segments, num_det;
    double ovthresh;
    const double *gt_corners, *det_corners;         /* DEVICE (num_gt, 8, 3), (num_det, 8, 3) */
    const double *det_scores;                       /* DEVICE (num_det) */
    const int32_t *det_segments;                    /* DEVICE (num_det) */
    const int32_t *gt_segment_offsets;              /* DEVICE (num_gt_segments + 1) */
    const int32_t *gt_class_offsets, *det_class_offsets;   /* DEVICE (num_classes + 1) */
    const int32_t *host_gt_segment_offsets, *host_gt_class_offsets, *host_det_class_offsets;   /* HOST copies */
    void *workspace;
    long long workspace_bytes;
    double *rec, *prec;                             /* DEVICE (num_det) */
    struct fcn_sunrgbd_eval_result_ *result;        /* DEVICE (num_classes) */
} fcn_sunrgbd_eval_args;
typedef struct fcn_sunrgbd_eval_result_ {
    double ap;
    int32_t npos, nd;                               /* ground-truth rows, detections of the class */
    int32_t status, reserved;
} fcn_sunrgbd_eval_result;
FCN_API long long fcn_sunrgbd_eval_workspace_bytes(const fcn_sunrgbd_eval_args *args);
FCN_API int fcn_sunrgbd_eval_match(const fcn_sunrgbd_eval_args *args, fcn_stream_t stream);
FCN_API int fcn_sunrgbd_eval_curves(const fcn_sunrgbd_eval_args *args, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (15) KITTI frustum extraction on the device: extract_frustum_data_rgb_detection of kitti/prepare_data.py:462-568
 *      (with kitti_util.py:172-210 and draw_util.py:12-23) for several frames and all their 2-D detections at once.
 *
 *      Per frame f (scan rows [scan_offsets[f], scan_offsets[f+1]) of `scans`, float32 x, y, z, intensity):
 *        ref  = V2C . [x, y, z, 1]   rect = R0 . ref   [u', v', w] = P . [rect, 1]   u = u' / w, v = v' / w
 *      in float64, every product and sum rounded separately, each row summed left to right (column 0 first).
 *      A point is in the image when 0 <= u < width, 0 <= v < height and x > 2 (NaN fails); those points are
 *      compacted per frame in scan order.
 *      Per detection d (frame det_frame[d], box xmin, ymin, xmax, ymax as read): the box clipped to [0, width-1] x
 *      [0, height-1]; its points are the frame's in-image points with xmin <= u < xmax and ymin <= v < ymax, in scan
 *      order; it is dropped when ymax - ymin < 5, xmax - xmin < 1 or it has no point.  The type whitelist is the
 *      caller's: pass only the detections of wanted types.  frustum_angle = -atan2(20, x) of project_image_to_rect
 *      of the clipped box centre at depth 20.
 *
 *      Two calls in order on one stream, sharing the caller's workspace (fcn_frustum_extract_workspace_bytes: needs the
 *      device, -1 on invalid arguments), no host sync, no allocation:
 *        fcn_frustum_extract_count : the in-image points, every detection's points, the drop rules and the prefix sums
 *                                    over the kept detections; writes det_points (DEVICE, num_dets: the detection's
 *                                    point count when kept, -1 when dropped or when det_frame is out of range) and
 *                                    info (DEVICE int64[4]: kept detections K, their points M, detections with an
 *                                    out-of-range frame, 0);
 *        fcn_frustum_extract_write : needs num_kept = K and num_out_points = M as read by the host; writes the kept
 *                                    detections in detection order: points (M, 4) float32 rect x, y, z and intensity,
 *                                    offsets (K + 1) int32, frustum_angle (K), box2d (K, 4) clipped, P (K, 12) the
 *                                    frame's P2, det_index (K) int32 index d.
 *      With num_frames == 0 or num_dets == 0 both calls return 0 and do nothing (K = M = 0; info is not written).
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    double P[12], V2C[12], R0[9];   /* P2 (3x4), Tr_velo_to_cam (3x4), R0_rect (3x3), row-major */
    int32_t height, width;          /* image size */
} fcn_frustum_frame;
typedef struct {
    int num_frames, num_points, num_dets, num_kept;
    long long num_out_points;
    const float *scans;                 /* DEVICE (num_points, 4), 16-byte aligned */
    const int32_t *scan_offsets;        /* DEVICE (num_frames + 1) */
    const int32_t *host_scan_offsets;   /* HOST copy: starts at 0, never decreases, ends at num_points */
    const fcn_frustum_frame *frames;    /* DEVICE (num_frames) */
    const double *boxes;                /* DEVICE (num_dets, 4) */
    const int32_t *det_frame;           /* DEVICE (num_dets) */
    void *workspace;
    long long workspace_bytes;
    long long *info;                    /* DEVICE int64[4] */
    int32_t *det_points;                /* DEVICE (num_dets) */
    float *points;                      /* fcn_frustum_extract_write outputs (DEVICE) */
    int32_t *offsets;
    double *frustum_angle, *box2d, *P;
    int32_t *det_index;
} fcn_frustum_extract_args;
FCN_API long long fcn_frustum_extract_workspace_bytes(const fcn_frustum_extract_args *args);
FCN_API int fcn_frustum_extract_count(const fcn_frustum_extract_args *args, fcn_stream_t stream);
FCN_API int fcn_frustum_extract_write(const fcn_frustum_extract_args *args, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (16) KITTI refinement frustums on the device: extract_frustum_data, extract_frustum_det_data and
 *      extract_frustum_data_rgb_detection of kitti/prepare_data_refine.py:239-773 for several frames and all their
 *      3-D boxes at once.
 *
 *      The frames' in-image points are those of section (15) (same projection, same test, scan order).  A job is one
 *      3-D box that cuts points out of its frame (job_frame[j]): the enlarged (and perhaps perturbed) box jobs[j].
 *      Every box is tested in float64 in its own frame: p in box <=> |cs dx - sn dz| <= half[0], |dy| <= half[1] and
 *      |sn dx + cs dz| <= half[2], with (dx, dy, dz) = p - center and every product and sum rounded separately.  The
 *      label box of a job (the points of the job that are also in it are labelled 1):
 *        FCN_REFINE_GT       gt_boxes[job_ref[j]]; the job is dropped when no point is labelled;
 *        FCN_REFINE_MATCHED  the ground truth matched to detection job_ref[j]: the first maximum of the 3-D IoU (the
 *                            reference's rbbox_iou_3d, float64, with its standup-box pre-filter at 0) of its corners
 *                            det_corners[d] against gt_corners[g] for the ground truths g in [gt_offsets[f],
 *                            gt_offsets[f + 1]) of its frame f = det_frame[d]; none when that maximum is below
 *                            iou_thresh.  The job is dropped without a match or when no point is labelled;
 *        FCN_REFINE_DET      none; the job is dropped when it has no point.
 *      num_pairs = sum over the detections of their frame's ground-truth count; pair_offsets is its exclusive sum.
 *
 *      Two calls in order on one stream, sharing the caller's workspace (fcn_refine_extract_workspace_bytes: needs the
 *      device, -1 on invalid arguments), no host sync, no allocation:
 *        fcn_refine_extract_count : writes job_points (DEVICE, num_jobs: the job's point count when kept, -1 when
 *                                   dropped or when an index is out of range), job_gt (DEVICE, num_jobs: the label
 *                                   box's index in gt_boxes, -1 for none) and info (DEVICE int64[4]: kept jobs K, their
 *                                   points M, jobs or detections with an out-of-range index, 0);
 *        fcn_refine_extract_write : needs num_kept = K and num_out_points = M as read by the host; writes the kept jobs
 *                                   in job order: points (M, 4) float32 rect x, y, z and intensity in scan order,
 *                                   labels (M) uint8 (not written in FCN_REFINE_DET mode; may be NULL) and offsets (K + 1)
 *                                   int32.  The k-th kept job is the k-th j with job_points[j] >= 0.
 *      With num_frames == 0 or num_jobs == 0 both calls return 0 and do nothing (K = M = 0; info is not written).
 * ------------------------------------------------------------------------------------------ */
#define FCN_REFINE_GT 0
#define FCN_REFINE_MATCHED 1
#define FCN_REFINE_DET 2
typedef struct {
    double center[3];   /* cx, cy - h / 2, cz (rect camera coordinates) */
    double half[3];     /* l / 2, h / 2, w / 2 */
    double cs, sn;      /* cos(ry), sin(ry) */
} fcn_refine_box;
typedef struct {
    int mode, num_frames, num_points, num_jobs, num_gt, num_dets, num_pairs, num_kept;
    long long num_out_points;
    double iou_thresh;
    const float *scans;                 /* DEVICE (num_points, 4), 16-byte aligned */
    const int32_t *scan_offsets;        /* DEVICE (num_frames + 1) */
    const int32_t *host_scan_offsets;   /* HOST copy: starts at 0, never decreases, ends at num_points */
    const fcn_frustum_frame *frames;    /* DEVICE (num_frames) */
    const fcn_refine_box *jobs;         /* DEVICE (num_jobs) */
    const int32_t *job_frame;           /* DEVICE (num_jobs) */
    const int32_t *job_ref;             /* DEVICE (num_jobs): ground-truth index (GT), detection index (MATCHED) */
    const fcn_refine_box *gt_boxes;     /* DEVICE (num_gt) */
    const double *gt_corners;           /* DEVICE (num_gt, 8, 3), MATCHED only */
    const double *det_corners;          /* DEVICE (num_dets, 8, 3), MATCHED only */
    const int32_t *det_frame;           /* DEVICE (num_dets), MATCHED only */
    const int32_t *gt_offsets;          /* DEVICE (num_frames + 1), MATCHED only */
    const int32_t *pair_offsets;        /* DEVICE (num_dets + 1), MATCHED only */
    void *workspace;
    long long workspace_bytes;
    long long *info;                    /* DEVICE int64[4] */
    int32_t *job_points, *job_gt;       /* DEVICE (num_jobs) each */
    float *points;                      /* fcn_refine_extract_write outputs (DEVICE) */
    uint8_t *labels;
    int32_t *offsets;
} fcn_refine_extract_args;
FCN_API long long fcn_refine_extract_workspace_bytes(const fcn_refine_extract_args *args);
FCN_API int fcn_refine_extract_count(const fcn_refine_extract_args *args, fcn_stream_t stream);
FCN_API int fcn_refine_extract_write(const fcn_refine_extract_args *args, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (17) KITTI first-stage training frustums on the device: the point work of extract_frustum_data and
 *      extract_frustum_det_data of kitti/prepare_data.py:102-391 (--gen_train, --gen_val and the _det extension) for
 *      several frames and all their jobs at once.
 *
 *      The frames' in-image points and their float64 image coordinates u, v are those of section (15) (same
 *      projection, same test, scan order).  A job j (jobs[j]) is one cutting 2-D box in frame jobs[j].frame and one
 *      label 3-D box label_boxes[jobs[j].label] (fcn_refine_box of section (16): centre (tx, ty - h/2, tz), half extents
 *      (l/2, h/2, w/2), ry; the corners of kitti_util.compute_box_3d).  The job's points are the frame's in-image
 *      points with u < xmax, u >= xmin, v < ymax and v >= ymin for the box as given (not clipped); a point is labelled
 *      1 when the section (16) half-space test puts it in the label box.  The job is dropped when no point is labelled.
 *      The perturbation, the 2-D matching and the 25-px rule are the caller's: pass only the jobs to cut.
 *
 *      Two calls in order on one stream, sharing the caller's workspace (fcn_gt_extract_workspace_bytes: needs the
 *      device, -1 on invalid arguments), no host sync, no allocation:
 *        fcn_gt_extract_count : writes job_points (DEVICE, num_jobs: the job's point count when kept, -1 when dropped
 *                               or when its frame or label index is out of range) and info (DEVICE int64[4]: kept jobs
 *                               K, their points M, jobs with an out-of-range index, 0);
 *        fcn_gt_extract_write : needs num_kept = K and num_out_points = M as read by the host; writes the kept jobs in
 *                               job order: points (M, 4) float32 rect x, y, z and intensity in scan order, labels (M)
 *                               uint8 and offsets (K + 1) int32.  The k-th kept job is the k-th j with
 *                               job_points[j] >= 0.
 *      With num_frames == 0 or num_jobs == 0 both calls return 0 and do nothing (K = M = 0; info is not written).
 * ------------------------------------------------------------------------------------------ */
typedef struct {
    double box[4];      /* cutting box xmin, ymin, xmax, ymax */
    int32_t frame;      /* index into frames */
    int32_t label;      /* index into label_boxes */
} fcn_gt_job;
typedef struct {
    int num_frames, num_points, num_jobs, num_labels, num_kept, reserved;
    long long num_out_points;
    const float *scans;                 /* DEVICE (num_points, 4), 16-byte aligned */
    const int32_t *scan_offsets;        /* DEVICE (num_frames + 1) */
    const int32_t *host_scan_offsets;   /* HOST copy: starts at 0, never decreases, ends at num_points */
    const fcn_frustum_frame *frames;    /* DEVICE (num_frames) */
    const fcn_gt_job *jobs;             /* DEVICE (num_jobs) */
    const fcn_refine_box *label_boxes;  /* DEVICE (num_labels) */
    void *workspace;
    long long workspace_bytes;
    long long *info;                    /* DEVICE int64[4] */
    int32_t *job_points;                /* DEVICE (num_jobs) */
    float *points;                      /* fcn_gt_extract_write outputs (DEVICE) */
    uint8_t *labels;
    int32_t *offsets;
} fcn_gt_extract_args;
FCN_API long long fcn_gt_extract_workspace_bytes(const fcn_gt_extract_args *args);
FCN_API int fcn_gt_extract_count(const fcn_gt_extract_args *args, fcn_stream_t stream);
FCN_API int fcn_gt_extract_write(const fcn_gt_extract_args *args, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (18) SUN-RGBD frustums on the device: the point work of extract_frustum_data and
 *      extract_frustum_data_from_rgb_detection of sunrgbd/prepare_data.py:132-381 (--gen_train, --gen_val,
 *      --gen_val_rgb_detection) for several frames and all their jobs at once.
 *
 *      Scans are (n, 6) float32 rows x, y, z, r, g, b in upright depth coordinates.  Every scan point is a candidate
 *      (no image-bounds test): its float64 image coordinates are project_upright_depth_to_image's, each np.dot
 *      accumulated as OpenBLAS's dgemm does (the first product rounded, then one FMA per further term) and the two
 *      divisions IEEE.  A job j (jobs[j], fcn_gt_job of section (17)) is one cutting 2-D box in frame jobs[j].frame
 *      and, when jobs[j].label >= 0, one label 3-D box label_boxes[jobs[j].label] (fcn_refine_box: centre
 *      (cx, -cz, cy), half extents (l, h, w), cs = cos(heading_angle), sn = sin(heading_angle), the corners of
 *      sunrgbd_utils.compute_box_3d flipped to upright camera coordinates).  Its in-box points are the frame's points
 *      with u < xmax, u >= xmin, v < ymax and v >= ymin, in scan order; a point is labelled 1 when the section (16)
 *      half-space test puts its upright camera coordinates (x, -z, y) in the label box.  labelled = 1 for the ground
 *      truth sets (all jobs have a label box), 0 for detections (no job has one).
 *
 *      Four calls in order on one stream, sharing the caller's workspace (fcn_sunrgbd_extract_workspace_bytes: needs
 *      the device, -1 on invalid arguments), no host sync, no allocation:
 *        fcn_sunrgbd_extract_project : u, v of every scan point into the workspace;
 *        fcn_sunrgbd_extract_count   : for the jobs [job_begin, job_end) (may run several times; the jobs of a
 *                                      range are uploaded before it, a later call overwrites a job's words):
 *                                      job_points (DEVICE, num_jobs: the in-box count n, -1 when the frame or
 *                                      label index is out of range) and job_labelled (DEVICE, num_jobs: its
 *                                      labelled points);
 *        fcn_sunrgbd_extract_select  : after every job is counted and the subsample draws uploaded: job_choice
 *                                      (DEVICE, num_jobs: c for the c-th job with n > 2048, -1 for the others),
 *                                      choice_ranks (DEVICE, num_choices x 2048: the in-box ranks np.random.choice
 *                                      chose, sorted) and choice_slots (DEVICE, same shape: the output row of each).
 *                                      A job keeps min(n, 2048) points; it is dropped when fewer than 5 of them are
 *                                      labelled (labelled = 1) or when n < 5 (labelled = 0).  Overwrites job_points
 *                                      with the kept count (-1 when dropped) and writes info (DEVICE
 *                                      int64[4]: kept jobs K, their points M, jobs with an out-of-range index, 0);
 *        fcn_sunrgbd_extract_write   : needs num_kept = K and num_out_points = M as read by the host; writes the kept
 *                                      jobs in job order: points (M, 6) float32 (x, -z, y, r, g, b), in scan order or,
 *                                      for a job with n > 2048, in choice order; labels (M) uint8 (labelled = 1
 *                                      only) and offsets (K + 1) int32.
 *      With num_frames == 0 or num_jobs == 0 every call returns 0 and does nothing (K = M = 0; info is not written).
 * ------------------------------------------------------------------------------------------ */
#define FCN_SUNRGBD_MAX_POINTS 2048
typedef struct {
    double Rtilt[9];    /* row-major */
    double K[9];        /* row-major */
} fcn_sunrgbd_frame;
typedef struct {
    int num_frames, num_points, num_jobs, num_labels, num_choices, labelled;
    int job_begin, job_end, num_kept, reserved;
    long long num_out_points;
    const float *scans;                 /* DEVICE (num_points, 6) */
    const int32_t *scan_offsets;        /* DEVICE (num_frames + 1) */
    const int32_t *host_scan_offsets;   /* HOST copy: starts at 0, never decreases, ends at num_points */
    const fcn_sunrgbd_frame *frames;    /* DEVICE (num_frames) */
    const fcn_gt_job *jobs;             /* DEVICE (num_jobs) */
    const fcn_refine_box *label_boxes;  /* DEVICE (num_labels) */
    const int32_t *job_choice;          /* DEVICE (num_jobs), select */
    const int32_t *choice_ranks;        /* DEVICE (num_choices, 2048), select and write */
    const int32_t *choice_slots;        /* DEVICE (num_choices, 2048), write */
    void *workspace;
    long long workspace_bytes;
    long long *info;                    /* DEVICE int64[4] */
    int32_t *job_points, *job_labelled; /* DEVICE (num_jobs) each */
    float *points;                      /* fcn_sunrgbd_extract_write outputs (DEVICE) */
    uint8_t *labels;
    int32_t *offsets;
} fcn_sunrgbd_extract_args;
FCN_API long long fcn_sunrgbd_extract_workspace_bytes(const fcn_sunrgbd_extract_args *args);
FCN_API int fcn_sunrgbd_extract_project(const fcn_sunrgbd_extract_args *args, fcn_stream_t stream);
FCN_API int fcn_sunrgbd_extract_count(const fcn_sunrgbd_extract_args *args, fcn_stream_t stream);
FCN_API int fcn_sunrgbd_extract_select(const fcn_sunrgbd_extract_args *args, fcn_stream_t stream);
FCN_API int fcn_sunrgbd_extract_write(const fcn_sunrgbd_extract_args *args, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (19) The evaluators' inputs from the detection collector's device rows: sections (13) and (14) fed from the rows of
 *      section (10) with no host pass over the rows.
 *
 *      rows / seg_offsets / keep_count are fcn_det_select's and fcn_det_prepare's outputs: kept row k of segment s is
 *      rows[seg_offsets[s] + k], k < keep_count[s].  The gather plan is per segment: seg_dst[s] is the output record of
 *      the segment's first kept row (its rows follow in row order), or -1 when the segment is not written;
 *      seg_value[s] is the KITTI type code (FCN_KITTI_*) or the SUN-RGBD ground-truth segment (or -1) of its rows.
 *      host_* are HOST copies, validated before anything is launched: seg_offsets start at 0, never decrease and end
 *      at num_rows, keep_count[s] fits its segment, every written segment stays inside [0, num_out) and their kept
 *      rows add up to num_out.  One launch (one thread per counted row), no host sync, no allocation, no workspace.
 *        fcn_det_kitti_records : records (num_out, FCN_KITTI_DET_COLS) of section (13): the type code, alpha =
 *                                compute_alpha(tx, tz, ry), box2d, h, w, l, tx, ty, tz, ry, each as '%.4f' then strtod
 *                                would give it, and the score as '%f' (exact: rint(x * 10^d) / 10^d in float64).
 *        fcn_det_sunrgbd_feed  : corners (num_out, 8, 3), scores (num_out) and segments (num_out) of section (14):
 *                                compute_box_3d's corners (float32 cos, sin and half sizes, float64 rotation and
 *                                translation, each operation rounded on its own), the float64 score and seg_value[s];
 *                                *status |= FCN_DET_FEED_NONFINITE (status may be NULL) when a score or corner is not
 *                                finite.
 *      atan2, cos and sin are computed in float64 and rounded once to float32 (the correctly rounded float32 value;
 *      numpy's float32 loops differ from it in the last bit on some inputs, depending on the CPU).
 * ------------------------------------------------------------------------------------------ */
#define FCN_DET_FEED_NONFINITE 1
typedef struct {
    int num_segments, num_rows, num_out, reserved0;
    const float *rows;                              /* DEVICE (num_rows, 12) */
    const int32_t *seg_offsets, *keep_count;        /* DEVICE (num_segments + 1), (num_segments) */
    const int32_t *seg_dst, *seg_value;             /* DEVICE (num_segments) each */
    const int32_t *host_seg_offsets, *host_keep_count, *host_seg_dst;   /* HOST copies */
    double *records;                                /* fcn_det_kitti_records: DEVICE (num_out, FCN_KITTI_DET_COLS) */
    double *corners, *scores;                       /* fcn_det_sunrgbd_feed: DEVICE (num_out, 8, 3), (num_out) */
    int32_t *segments;                              /* fcn_det_sunrgbd_feed: DEVICE (num_out) */
    int32_t *status;                                /* fcn_det_sunrgbd_feed: DEVICE int32, optional */
} fcn_det_eval_feed_args;
FCN_API int fcn_det_kitti_records(const fcn_det_eval_feed_args *args, fcn_stream_t stream);
FCN_API int fcn_det_sunrgbd_feed(const fcn_det_eval_feed_args *args, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (20) The refinement stage's inputs from the detection collector's device rows: the jobs of section (16) in
 *      FCN_REFINE_DET or FCN_REFINE_MATCHED mode and the kept frustums' lists and fcn_train_frustum records of section
 *      (11), with no host pass over the rows (kitti/prepare_data_refine.py --gen_val_det / --gen_from_folder fed from
 *      the collector instead of result files).
 *
 *      The gather plan is per piece: piece p is the kept rows [piece_row[p], piece_row[p] + n_p) of one collector
 *      segment (section (19)'s rows), n_p = piece_offsets[p + 1] - piece_offsets[p]; job piece_offsets[p] + i is row
 *      piece_row[p] + i, in frame piece_frame[p] (an index into section (16)'s frames), image piece_image[p], class
 *      index piece_class[p] (the fcn_train_frustum cls_index).  The host builds the plan from segment metadata alone,
 *      in the job order of the dict path: the images of image_ids, then the collector's classes of each image in its
 *      dict order (whitelisted ones only), then the rows.  host_piece_offsets / host_piece_row are HOST copies,
 *      validated before anything is launched.  One launch each, no host sync, no allocation, no workspace.
 *        fcn_refine_jobs_from_rows    one thread per job.  The row read back as its '%.4f' / '%f' text (section (19)'s
 *                                     quantization), the box array a = [tx, ty - h/2, tz, l, w, h, ry] in float64,
 *                                     every operation rounded on its own; status[j] |= FCN_REFINE_ROW_NONFINITE when a
 *                                     is not finite, FCN_REFINE_ROW_EXTENTS when l, w or h is not positive, and in
 *                                     FCN_REFINE_DET mode FCN_REFINE_ROW_DROPPED when ymax - ymin < 5 or xmax - xmin < 1
 *                                     (the quantized 2-D box).  jobs[j]: the box enlarged x1.2 (centre, half extents,
 *                                     cos / sin of ry); a bad or dropped job of FCN_REFINE_DET mode gets half extents
 *                                     -1, so section (16)'s count pass keeps none of its points and drops it.
 *                                     job_frame[j] = piece_frame, job_ref[j] = j; FCN_REFINE_MATCHED: det_corners[j]
 *                                     (8, 3), rbbox_iou_3d's corners of a (not enlarged).  job_data[j]: the enlarged
 *                                     box array, the quantized 2-D box and score, image and class index.
 *        fcn_refine_frustum_table     after section (16)'s count pass, one thread per kept job kept[k]: lists (num_kept,
 *                                     FCN_REFINE_LIST_COLS) float64: frustum_angle -atan2(cz, cx), the 24 corners of
 *                                     compute_box_3d_obj_array (np.dot's dgemm order: the first product rounded, then
 *                                     one FMA per term), the 3 sizes, the angle, the 2-D box, the score; records
 *                                     (num_kept, zeroed by the caller): the refine fields of section (11) - rot, cs,
 *                                     sn, ref_center, line0, line_delta, z_start, z_step and T for stride[0 ..
 *                                     num_scales), cls_index and, when labels, the matched ground truth's terms
 *                                     gt_terms[job_gt[j]] in the predicted box's frame, else rgb_prob = the score;
 *                                     words (num_kept, num_scales + 1) int32: T per scale, then 1 when the predicted
 *                                     box is degenerate (a T below 1 or a zero line), else 0.
 *      cos, sin and atan2 are CUDA's float64 functions (within 2 ulp); everything else follows numpy's expressions.
 * ------------------------------------------------------------------------------------------ */
#define FCN_REFINE_ROW_NONFINITE 1
#define FCN_REFINE_ROW_EXTENTS 2
#define FCN_REFINE_ROW_DROPPED 4
#define FCN_REFINE_LIST_COLS 34   /* frustum_angle, pred_box3d (24), pred_box3d_size (3), pred_box3d_angle, box2d (4), prob */
typedef struct {
    double cut[7];      /* enlarged box array [tx, ty - h/2, tz, 1.2 l, 1.2 w, 1.2 h, ry] */
    double box2d[4];    /* quantized x1, y1, x2, y2 */
    double prob;        /* quantized score */
    int32_t image, cls_index;
} fcn_refine_job_data;
typedef struct {
    double center[3];   /* (box3d[0] + box3d[6]) / 2 of the ground truth's compute_box_3d_obj_array corners */
    double heading;     /* ry */
    double size[3];     /* l, w, h */
    double dist;        /* sqrt(l^2 + w^2) */
} fcn_refine_gt_terms;
typedef struct {
    int mode, num_pieces, num_jobs, num_rows;
    const float *rows;                              /* DEVICE (num_rows, 12), the collector's rows */
    const int32_t *piece_offsets;                   /* DEVICE (num_pieces + 1) */
    const int32_t *piece_row, *piece_frame, *piece_image, *piece_class;   /* DEVICE (num_pieces) each */
    const int32_t *host_piece_offsets, *host_piece_row;                    /* HOST copies */
    fcn_refine_box *jobs;                           /* DEVICE (num_jobs) outputs */
    int32_t *job_frame, *job_ref, *status;
    double *det_corners;                            /* DEVICE (num_jobs, 8, 3), FCN_REFINE_MATCHED only */
    fcn_refine_job_data *job_data;
} fcn_refine_jobs_args;
typedef struct {
    int mode, labels, num_kept, num_jobs, num_gt, num_scales;
    double stride[FCN_MAX_SCALES];
    const int32_t *kept;                            /* DEVICE (num_kept): the job of each kept frustum */
    const int32_t *job_gt;                          /* DEVICE (num_jobs): section (16)'s job_gt, labels only */
    const fcn_refine_job_data *job_data;            /* DEVICE (num_jobs) */
    const fcn_refine_gt_terms *gt_terms;            /* DEVICE (num_gt), labels only */
    double *lists;                                  /* DEVICE (num_kept, FCN_REFINE_LIST_COLS) */
    fcn_train_frustum *records;                     /* DEVICE (num_kept) */
    int32_t *words;                                 /* DEVICE (num_kept, num_scales + 1) */
} fcn_refine_frustum_table_args;
FCN_API int fcn_refine_jobs_from_rows(const fcn_refine_jobs_args *args, fcn_stream_t stream);
FCN_API int fcn_refine_frustum_table(const fcn_refine_frustum_table_args *args, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (21) Frame detection in fixed capacities: sections (15), (9) and (10) for F frames of at most P scan points and D
 *      2-D detections each, with every size read on the device.  No host sync, no allocation: a call can be captured
 *      in a CUDA graph and replayed on new frames written into the same buffers.
 *
 *      fcn_frame_extract : section (15) over the F * D detection slots (slot f * D + j is detection j of frame f).
 *        Frame f holds min(scan_counts[f], P) points (rows [f * P, f * P + n) of scans) and min(det_counts[f], D)
 *        detections; a detection is a candidate when bit det_class[d] (0 Car, 1 Pedestrian, 2 Cyclist) is set in
 *        class_mask.  The count pass is section (15)'s; each frame's kept frustums then share P_out = out_capacity
 *        points: a kept frustum whose points would end past the frame's P_out (counting every kept frustum before it
 *        in the frame) is dropped, so no store is cut short.  The write pass is section (15)'s.  Outputs, over B = F * D batch entries: the kept frustums first in slot
 *        order, then B - K dummy entries (one point at the origin, angle 0, box (0, 0, 1, 1), a unit P).
 *          points (F * P_out + B, 4)   offsets (B + 1)   frustum_angle (B)   box2d (B, 4)   P (B, 12)
 *          det_index (B): the slot, -1 for a dummy      valid (B): 1 for a kept frustum
 *          cls_index (B): det_class of the slot         rgb_prob (B): det_prob of the slot (float32)
 *          seg (B): f * 3 + r, r the rank of the frustum's class among its frame's kept classes by first appearance
 *            (the classes of the frustums in the batch: one dropped for P_out gives its class no rank)
 *          seg_class (F * 3): the class of segment f * 3 + r, -1 when the frame has fewer kept classes
 *        *status gets FCN_FRAME_* bits OR-ed in (the caller clears it).
 *      fcn_resample_choice : the (B, N) int32 `choice` of section (9), one CTA per entry b with n = offsets[b+1] -
 *        offsets[b] points.  n >= N: N distinct indices in random order (the N smallest of one 40-bit key per point,
 *        ties by index, ordered by key); 0 < n < N: N indices drawn uniformly with replacement.  The draws are
 *        Philox4x32-10 with key (seed low, seed high) and counter (i, det_index[b], *call low, *call high); an entry
 *        with det_index -1 uses B + b.  n <= 0 writes zeros.  Needs N <= 2048 and n < 2^24.
 *      fcn_det_candidates_valid : fcn_det_candidates where entry b adds no row unless valid[b] != 0.
 *      fcn_det_finalize_capacity : fcn_det_prepare and fcn_det_select in one call, with the row count and the bit-matrix
 *        offsets read on the device: n = min(*counter, capacity), `mask` of mask_words words must hold every segment's
 *        bit matrix (mask_words >= capacity * ceil(m / 32), m the most rows one segment can hold); n_counted is ignored.
 *        ORs FCN_FRAME_ROWS into *status when *counter > capacity (the rows past it were not recorded).
 * ------------------------------------------------------------------------------------------ */
#define FCN_FRAME_SCAN_POINTS 1     /* a frame had more than P scan points (the first P were used) */
#define FCN_FRAME_DETS 2            /* a frame had more than D detections (the first D were used) */
#define FCN_FRAME_OUT_POINTS 4      /* a frame's kept frustums had more than P_out points (dropped as above) */
#define FCN_FRAME_ROWS 8            /* more candidate rows than the collector's capacity R */
#define FCN_FRAME_BAD_DET 16        /* a detection with a class outside 0..2 or a non-finite box (not extracted) */
typedef struct {
    int num_frames, scan_capacity, det_capacity, out_capacity;   /* F, P, D, P_out */
    uint32_t class_mask;
    const float *scans;                 /* DEVICE (F * P, 4), 16-byte aligned */
    const int32_t *scan_counts;         /* DEVICE (F) */
    const fcn_frustum_frame *frames;    /* DEVICE (F) */
    const double *boxes;                /* DEVICE (F * D, 4) */
    const int32_t *det_class;           /* DEVICE (F * D) */
    const float *det_prob;              /* DEVICE (F * D) */
    const int32_t *det_counts;          /* DEVICE (F) */
    void *workspace;
    long long workspace_bytes;
    int32_t *status;                    /* DEVICE scalar */
    float *points;                      /* outputs (DEVICE), see above */
    int32_t *offsets;
    double *frustum_angle, *box2d, *P;
    int32_t *det_index, *valid, *cls_index, *seg, *seg_class;
    float *rgb_prob;
} fcn_frame_extract_args;
FCN_API long long fcn_frame_extract_workspace_bytes(const fcn_frame_extract_args *args);
FCN_API int fcn_frame_extract(const fcn_frame_extract_args *args, fcn_stream_t stream);
typedef struct {
    int B, N;
    unsigned long long seed;
    const int32_t *offsets;             /* DEVICE (B + 1) */
    const int32_t *det_index;           /* DEVICE (B) */
    const long long *call;              /* DEVICE scalar: the call counter */
    int32_t *choice;                    /* DEVICE (B, N) */
} fcn_resample_args;
FCN_API int fcn_resample_choice(const fcn_resample_args *args, fcn_stream_t stream);
FCN_API int fcn_det_candidates_valid(const fcn_det_candidate_args *args, const int32_t *valid, fcn_stream_t stream);
FCN_API int fcn_det_finalize_capacity(const fcn_det_finalize_args *args, int32_t *status, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (22) Frame refinement in fixed capacities: sections (20), (16) and (11) for the result of one section (21) call,
 *      with every size read on the device, so the refinement stage joins the detection stage in one CUDA graph.
 *
 *      fcn_frame_refine_extract : the refinement frustums of F frames, J jobs a frame (slot f * J + j), from the first
 *        stage's rows (num_rows, 12), seg_offsets (3F + 1), keep_count (3F) and seg_class (F, 3), and the scans,
 *        scan counts and frames the first stage read (frames of at most P = scan_capacity points).
 *        Jobs: frame f's jobs are the kept rows of its segments 3f + r whose class seg_class[f, r] is set in
 *          class_mask, in r order, rows k < keep_count in order (the dict path's job order); rows past J set
 *          FCN_FRAME_JOBS and are not used.  Each job is section (20)'s FCN_REFINE_DET job (rj_jobs_kernel itself): the
 *          row's text quantization, the x1.2 enlargement and the silent ymax - ymin < 5 / xmax - xmin < 1 drop; a row
 *          with a non-finite box or a non-positive extent is dropped and sets FCN_FRAME_BAD_DET.
 *        Points: the frames' in-image points (section (15)'s, recomputed here from the scans), then section (16)'s
 *          count and write passes over the F * J slots.
 *        Slots: a frustum whose record needs more sections than widths[s] at any scale s is dropped and sets
 *          FCN_FRAME_SECTIONS; of the others, each frame's frustums fit, in slot order, while the frame's running
 *          point count stays <= P2_out = out_capacity; a frustum past it is dropped whole (so is every later one of the
 *          frame) and sets FCN_FRAME_OUT_POINTS.
 *        Outputs, over B2 = F * J batch entries: the kept frustums first in slot order, then B2 - K dummy entries (one
 *          point at the origin, a finite record with T[s] = 1, valid 0, box (0, 0, 1, 1)).
 *          points (F * P2_out + B2, 4)   offsets (B2 + 1)   job_index (B2): the slot, -1 for a dummy
 *          valid (B2)   cls_index (B2): the row's class   box2d (B2, 4) float32: the row's 2-D box as read back
 *          seg (B2): 3 f + r, r the rank of the frustum's class among its frame's kept frustums by first appearance
 *          seg_class_out (F * 3): the class of segment 3 f + r, -1 when the frame has fewer kept classes
 *          records (B2): section (20)'s fcn_train_frustum records (fcn_refine_frustum_table, labels 0) for stride[0 ..
 *            num_scales): rgb_prob is the row's score as read back.
 *        *status gets FCN_FRAME_* bits OR-ed in (the caller sets it).  No store lands outside a buffer whatever the
 *        inputs: rows outside [0, num_rows) are not read.
 *      fcn_build_train_inputs_fixed : fcn_build_train_inputs (section (11)) with each scale's collate width widths[s]
 *        (HOST, num_scales values >= 1) instead of the batch's largest T[s]; centers[s] is (B, 3, widths[s]) and columns
 *        >= T[s] of an item repeat its last column (collate_fn's mode='edge'); an item with T[s] > widths[s] is cut.
 * ------------------------------------------------------------------------------------------ */
#define FCN_FRAME_JOBS 32           /* a frame had more than J whitelisted first-stage rows (the first J were used) */
#define FCN_FRAME_SECTIONS 64       /* a refinement frustum needed more sections than W[s] (dropped) */
typedef struct {
    int num_frames, scan_capacity, job_capacity, out_capacity;   /* F, P, J, P2_out */
    int num_rows, num_scales;                                    /* R of the first stage, S */
    uint32_t class_mask;
    int reserved;
    double stride[FCN_MAX_SCALES];
    int32_t widths[FCN_MAX_SCALES];     /* W[s] */
    const float *scans;                 /* DEVICE (F * P, 4), 16-byte aligned */
    const int32_t *scan_counts;         /* DEVICE (F) */
    const fcn_frustum_frame *frames;    /* DEVICE (F) */
    const float *rows;                  /* DEVICE (num_rows, 12): the first stage's rows */
    const int32_t *seg_offsets;         /* DEVICE (3F + 1) */
    const int32_t *keep_count;          /* DEVICE (3F) */
    const int32_t *seg_class;           /* DEVICE (F * 3) */
    void *workspace;
    long long workspace_bytes;
    int32_t *status;                    /* DEVICE scalar */
    float *points;                      /* outputs (DEVICE), see above */
    int32_t *offsets, *job_index, *valid, *cls_index, *seg, *seg_class_out;
    fcn_train_frustum *records;
    float *box2d;
} fcn_frame_refine_args;
FCN_API long long fcn_frame_refine_extract_workspace_bytes(const fcn_frame_refine_args *args);
FCN_API int fcn_frame_refine_extract(const fcn_frame_refine_args *args, fcn_stream_t stream);
FCN_API int fcn_build_train_inputs_fixed(const fcn_train_input_args *args, const int32_t *widths,
                                         fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (23) SUN-RGBD frame extraction in fixed capacities: section (18)'s from_rgb_detection set (prepare_data.py:270-381)
 *      for F frames of at most P cloud points and D 2-D detections each, with every size read on the device and the
 *      2048-point cap drawn there.  No host sync, no allocation: a call can be captured in a CUDA graph.
 *
 *      fcn_sunrgbd_frame_extract : slot f * D + j is detection j of frame f.  Frame f holds min(cloud_counts[f], P)
 *        points (rows [f * P, f * P + n) of clouds: x, y, z, r, g, b in upright depth coordinates) and
 *        min(det_counts[f], D) detections; counts below 0 read as 0.  A detection is a candidate when its class
 *        det_class (an index into SUNRGBD_CLASSES, 0..9) is set in class_mask and its box is finite; a class outside
 *        0..9 or a non-finite box sets FCN_FRAME_BAD_DET.
 *        In-box points: section (18)'s, u < xmax, u >= xmin, v < ymax, v >= ymin of the float64 projection, in scan
 *          order (the rank of a point among its slot's in-box points is its scan-order rank).  A slot with n < 5
 *          in-box points is dropped (prepare_data.py:352).
 *        Cap: for every candidate with n > 2048, cap_choice[slot] holds 2048 distinct in-box ranks in random order,
 *          fcn_resample_choice's n >= N draw (N = 2048) keyed on (seed, *call, slot): np.random.choice(n, 2048,
 *          replace=False) of the reference.  The frustum keeps those points in that order; other rows of cap_choice
 *          are 0.  The caller keeps *call apart from its other draws' counters and advances it per call.
 *        Budget: each frame's kept frustums share P_out = out_capacity points, counting min(n, 2048) per frustum in
 *          slot order; a frustum past the budget is dropped whole (so is every later one of the frame) and sets
 *          FCN_FRAME_OUT_POINTS.
 *        Outputs, over B = F * D batch entries: the kept frustums first in slot order, then B - K dummy entries (one
 *          point at the origin, a finite record, valid 0, box (0, 0, 1, 1)).
 *          points (F * P_out + B, 6): x, -z, y, r, g, b     xyz (F * P_out + B, 3): the first three columns
 *          offsets (B + 1)   det_index (B): the slot, -1 for a dummy   valid (B)   cls_index (B): det_class
 *          rgb_prob (B): det_prob   box2d (B, 4) float32: the detection's box
 *          seg (B): 10 f + r, r the rank of the frustum's class among its frame's kept frustums by first appearance
 *          seg_class (F * 10): the class of segment 10 f + r, -1 when the frame has fewer kept classes
 *          records (B): the fcn_train_frustum of FCN_TRAIN_SUNRGBD, labels = 0: rot = pi / 2 + frustum_angle (the box
 *            centre at depth 20 through project_image_to_upright_camera, Rtilt @ in dgemm order, then -atan2(z, x);
 *            atan2, cos and sin are CUDA's float64 functions, within 2 ulp), cs, sn, cx, cy, K, Rtilt, rgb_prob,
 *            cls_index and T[s] = len(np.arange(0, max_depth, stride[s])) for s < num_scales, dummies included.
 *        *status gets FCN_FRAME_* bits OR-ed in (the caller clears it).  No store lands outside a buffer whatever the
 *        inputs.  Needs 1 <= D <= 64 (each point carries one in-box bit per detection of its frame).
 * ------------------------------------------------------------------------------------------ */
#define FCN_SUNRGBD_FRAME_CLASSES 10
#define FCN_SUNRGBD_FRAME_MAX_DETS 64
typedef struct {
    int num_frames, point_capacity, det_capacity, out_capacity;   /* F, P, D, P_out */
    uint32_t class_mask;                /* bit c: SUNRGBD_CLASSES[c] */
    int num_scales;
    unsigned long long seed;            /* the cap draw's key */
    double max_depth;
    double stride[FCN_MAX_SCALES];
    const float *clouds;                /* DEVICE (F * P, 6), 4-byte aligned */
    const int32_t *cloud_counts;        /* DEVICE (F) */
    const fcn_sunrgbd_frame *frames;    /* DEVICE (F) */
    const double *boxes;                /* DEVICE (F * D, 4) */
    const int32_t *det_class;           /* DEVICE (F * D) */
    const float *det_prob;              /* DEVICE (F * D) */
    const int32_t *det_counts;          /* DEVICE (F) */
    const long long *call;              /* DEVICE scalar: the cap draw's call counter */
    void *workspace;
    long long workspace_bytes;
    int32_t *status;                    /* DEVICE scalar */
    float *points, *xyz;                /* outputs (DEVICE), see above */
    int32_t *offsets, *det_index, *valid, *cls_index, *seg, *seg_class;
    float *rgb_prob, *box2d;
    int32_t *cap_choice;                /* DEVICE (B, 2048) */
    fcn_train_frustum *records;         /* DEVICE (B) */
} fcn_sunrgbd_frame_extract_args;
FCN_API long long fcn_sunrgbd_frame_extract_workspace_bytes(const fcn_sunrgbd_frame_extract_args *args);
FCN_API int fcn_sunrgbd_frame_extract(const fcn_sunrgbd_frame_extract_args *args, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (24) SUN-RGBD depth clouds: the SUNRGBD toolbox's read3dPoints as the reference's port restates it
 *      (sunrgbd/read_3d_points.py), for F depth images of at most H x W pixels, into section (23)'s `clouds` input.
 *      No host sync, no allocation: a call can be captured in a CUDA graph.
 *
 *      fcn_sunrgbd_depth_cloud : frame f is the top-left min(h, H) x min(w, W) crop of depth[f] (h, w = image_hw[f];
 *        values below 0 read as 0); pixel (v, u) is depth[f, v, u], 0-based row v and column u.
 *        Per pixel, with raw = depth[f, v, u]: a pixel is valid when raw != 0;
 *          r = (raw >> 3) | (raw << 13) in uint16 (a rotate right by 3), d = min(float(r) / 1000, 8) in float32;
 *          x3 = ((u - cx) * d) / fx, y3 = ((v - cy) * d) / fy in float64 (cx = K[0, 2], cy = K[1, 2], fx = K[0, 0],
 *          fy = K[1, 1]); the point (x3, d, -y3) times Rtilt in float64, each row as np.matmul(Rtilt, points.T) sums it
 *          (dgemm's a0 b0 rounded, then one FMA per further term; a frame of exactly one valid pixel goes through
 *          gemv instead: a1 b1 rounded, then FMAs of term 0 and term 2), rounded to float32 once;
 *          r, g, b = float(rgb[f, v, u, c]) / 255 in float32, or 0 when rgb is NULL.
 *        Outputs: clouds[f, k] (x, y, z, r, g, b) for the k-th valid pixel of the frame in row-major order, k < P;
 *          counts[f] = min(valid pixels, P).  Rows at and past counts[f] are not written.
 *        *status gets bits OR-ed in (the caller clears it): FCN_FRAME_SCAN_POINTS when a frame has more than P valid
 *        pixels (the first P are kept, in order), FCN_FRAME_PIXELS when h > H or w > W (the crop is read).
 *        No store lands outside a buffer whatever the inputs.
 * ------------------------------------------------------------------------------------------ */
#define FCN_FRAME_PIXELS 128        /* an image larger than the H x W capacity (its top-left H x W crop was read) */
typedef struct {
    int num_frames, height, width, point_capacity;   /* F, H, W, P */
    const uint16_t *depth;              /* DEVICE (F, H, W), 2-byte aligned */
    const uint8_t *rgb;                 /* DEVICE (F, H, W, 3) in RGB order, or NULL */
    const int32_t *image_hw;            /* DEVICE (F, 2): h, w of each frame */
    const double *calibs;               /* DEVICE (F, 18): Rtilt, then K, row-major, 8-byte aligned */
    void *workspace;
    long long workspace_bytes;
    int32_t *status;                    /* DEVICE scalar */
    float *clouds;                      /* DEVICE (F, P, 6), 4-byte aligned */
    int32_t *counts;                    /* DEVICE (F) */
} fcn_sunrgbd_depth_args;
FCN_API long long fcn_sunrgbd_depth_cloud_workspace_bytes(const fcn_sunrgbd_depth_args *args);
FCN_API int fcn_sunrgbd_depth_cloud(const fcn_sunrgbd_depth_args *args, fcn_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * (25) Frame detection store: the kept rows of many section (21), (22) or (23) calls appended to one device table, so
 *      a split run through a captured CUDA graph is scored or refined from one read.  Every size is read on the
 *      device: an append is captured in the same graph as the call it stores.
 *
 *      fcn_frame_store_append : one call's result, rows (num_rows, 12), seg_offsets (S + 1), keep_count (S) and
 *        seg_class (F, C) with S = C * F (segment s = C f + r), its status word, and ids (F): the image id of frame
 *        slot f, negative for a slot that contributes nothing.  The call's segments are those with seg_class >= 0 and
 *        ids[f] >= 0, in s order (frame slot, then class by first appearance), zero-keep segments included; segment
 *        s's rows are [seg_offsets[s], seg_offsets[s] + keep_count[s]) cut to [0, num_rows).
 *        A call is stored whole or not at all.  With n segments and m rows, when cursor->segments + n <=
 *        segment_capacity and cursor->rows + m <= row_capacity, the call's j-th segment becomes store segment
 *        d = cursor->segments + j: store_image[d] = ids[f], store_class[d] = seg_class[s], store_frame[d] =
 *        cursor->calls * F + f (mod 2^32), store_offset[d] = its first store row, store_keep[d] = its rows; then
 *        store_offset[cursor->segments + n] = cursor->rows + m, the rows are copied bit for bit, the cursor's
 *        segments and rows advance, calls grows by one and frame_status |= *status.  Otherwise nothing of the call is
 *        written and cursor->status gets FCN_STORE_SEGMENTS and / or FCN_STORE_ROWS.  Earlier calls stay intact, and
 *        no store lands outside a buffer whatever the call's tables hold.  The cursor starts zeroed; appends on one
 *        stream are ordered and nothing else writes the store meanwhile.
 * ------------------------------------------------------------------------------------------ */
#define FCN_STORE_ROWS 1            /* a call's rows did not fit the store's row capacity (the call was not stored) */
#define FCN_STORE_SEGMENTS 2        /* a call's segments did not fit the segment capacity (the call was not stored) */
#define FCN_STORE_MAX_FRAMES 65535
#define FCN_STORE_MAX_CLASSES 64
typedef struct {
    int32_t segments, rows;             /* store segments and rows used */
    int32_t calls;                      /* calls stored */
    int32_t status;                     /* FCN_STORE_* bits */
    int32_t frame_status;               /* OR of the stored calls' FCN_FRAME_* words */
} fcn_frame_store_cursor;
typedef struct {
    int num_frames, num_classes, num_rows;          /* F, C and the row capacity R of the appended call */
    int row_capacity, segment_capacity;             /* the store's */
    int reserved;
    const float *rows;                  /* DEVICE (num_rows, 12), 16-byte aligned */
    const int32_t *seg_offsets;         /* DEVICE (S + 1) */
    const int32_t *keep_count;          /* DEVICE (S) */
    const int32_t *seg_class;           /* DEVICE (F, C) */
    const int32_t *status;              /* DEVICE scalar: the call's FCN_FRAME_* word */
    const int64_t *ids;                 /* DEVICE (F) */
    void *workspace;
    long long workspace_bytes;
    float *store_rows;                  /* DEVICE (row_capacity, 12), 16-byte aligned */
    int64_t *store_image;               /* DEVICE (segment_capacity) */
    int32_t *store_class, *store_frame; /* DEVICE (segment_capacity) */
    int32_t *store_offset;              /* DEVICE (segment_capacity + 1) */
    int32_t *store_keep;                /* DEVICE (segment_capacity) */
    fcn_frame_store_cursor *cursor;     /* DEVICE */
} fcn_frame_store_args;
FCN_API long long fcn_frame_store_append_workspace_bytes(const fcn_frame_store_args *args);
FCN_API int fcn_frame_store_append(const fcn_frame_store_args *args, fcn_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* FRUSTUM_B200_H_ */
