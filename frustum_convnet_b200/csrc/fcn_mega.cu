// Persistent FCN kernel: ALL conv / transposed-conv / merge layers of ConvFeatNet, the two heads and the eval
// decode of one forward in ONE launch (replaces the 14 fcn_conv_gemm launches + fcn_decode_eval;
// reference models/det_base.py:196-224,367-411).
//
// Why: every per-layer launch pays a fixed cost per CTA (launch/PDL wait, barrier set-up, pipeline fill, drain)
// for a few microseconds of tensor-core work on grids of 9-72 CTAs.
//
// Design
//   * work unit ("job") = one [128 rows x NT columns] output tile of one layer; the host builds the job table in
//     TOPOLOGICAL order (every job depends only on jobs with a smaller index);
//   * persistent CTAs fetch the next job with ONE atomicAdd (dynamic scheduling).  Together with the topological
//     order this is deadlock-free under ANY co-residency: the smallest unfinished job is always owned by a running
//     CTA whose dependencies are complete - no grid-wide barrier, no co-residency requirement, late CTAs
//     (several forwards are in flight on other streams) simply pick up what is left;
//   * layer-to-layer dependencies are per row tile: a finished tile publishes a counter (release, gpu scope); the
//     scheduler warp acquires the counters of the (<= 4) source tiles a job reads (taps +-1, stride 2,
//     pixel-shuffled transposed convs) one job ahead, the TMA producer then crosses to the async proxy;
//   * inside a CTA the same warp-specialised pipeline as conv_gemm_tma.cu, made continuous across jobs: warp 9 =
//     scheduler (job fetch, descriptor, dependency polling), warp 8 = TMA producer (A boxes by cp.async.bulk.tensor
//     with the conv taps / stride in the coordinates, weight atoms and the job's bias slice by bulk copies),
//     warps 0-7 = two consumer warpgroups (wgmma, 64 rows each, N = NT = 256 | 128 | 64), warp 10 = store warp;
//     the smem stage ring of 32-wide K atoms runs across job boundaries (the next job's operands stream while the
//     current one is still multiplied or stored);
//   * epilogue off the tensor-core path: a consumer warpgroup adds the bias (from shared memory), applies ReLU and
//     TF32 rounding, writes zeros at pad positions and stages the result in its own [64 rows x 128 columns] buffer
//     (128-byte swizzled [32 x 32] boxes of the layer's store map, conflict-free fragment writes), arrives on
//     `staged` and goes straight into the next job's K loop.  The store warp stores the boxes by
//     cp.async.bulk.tensor (the transposed convs' pixel shuffle and the concat offset are in the map coordinates,
//     rows past the map are clipped), hands the buffer back (`staging_free`) once the bulk reads are done, waits
//     for the writes, crosses from the async proxy (fence.proxy.async.global) and publishes ONE count per tile
//     (red.release.gpu).  NT = 256 passes through the buffer in two 128-column halves.  The store warp waits only
//     on its own CTA's job queue and consumers and on its own bulk groups, so the argument above still holds;
//   * the heads tile (NT = 64: all 2 + 39 logits of a position) stores the logits row and decodes it
//     (decode.cuh - the same function the stand-alone decode kernel uses), writing the 6-tuple to the local
//     result block AND to the peers' gather buffers over NVLink (multi-GPU: no NCCL all-gather, no extra
//     launch; one epoch flag per forward);
//   * self-cleaning: the last CTA to finish resets the job counter and the tile flags for the next forward.
#include <cuda.h>

#include "common.cuh"
#include "decode.cuh"
#include "wgmma.cuh"

namespace fcn {
using namespace gmma;

constexpr int MG_ROWS = 128;
constexpr int MG_MMA_WARPS = 8;      // warps 0-7: two consumer warpgroups (MMA + staging of the epilogue)
constexpr int MG_TMA_WARP = MG_MMA_WARPS, MG_SCHED_WARP = MG_MMA_WARPS + 1, MG_STORE_WARP = MG_MMA_WARPS + 2;
constexpr int MG_THREADS = (MG_MMA_WARPS + 3) * 32;
constexpr int MG_SMEM_LIMIT = 232448;                         // 227 KB of dynamic shared memory per CTA
// Epilogue staging: per consumer warpgroup 64 rows x 128 fp32 columns as eight 128-byte-swizzled [32 x 32] boxes of
// the store map, box (column block cb, row block rb) at (2 cb + rb) * 4 KB.
constexpr int MG_STG_COLS = 128, MG_BOX_BYTES = 32 * 128, MG_STG_BYTES = 64 * MG_STG_COLS * 4;
constexpr int MG_A_ATOM = MG_ROWS * 128;
constexpr int MG_MAX_SLOTS = 8;
constexpr int MG_JOBQ = 4;                                    // job descriptors in flight inside a CTA
// full/empty, job_full/job_empty, taken, staged[2], staging_free[2]
constexpr int MG_NBAR = 2 * MG_MAX_SLOTS + 2 * MG_JOBQ + 1 + 4;
constexpr int MG_OFF_BAR = 2 * MG_STG_BYTES;
// barriers and the last-CTA flag, then fcn_mega_job[MG_JOBQ] (64 B each)
constexpr int MG_OFF_JOBQ = MG_OFF_BAR + ((MG_NBAR * 8 + 4 + 63) & ~63);
constexpr int MG_BIAS_FLOATS = 256;                          // bias slice of one queued job (NT <= 256 columns)
constexpr int MG_OFF_BIAS = MG_OFF_JOBQ + MG_JOBQ * 64;
constexpr int MG_OFF_RING = (MG_OFF_BIAS + MG_JOBQ * MG_BIAS_FLOATS * 4 + 1023) & ~1023;
// Stage ring: every stage carries ONE 32-wide K atom, a slot = [128 x 32] A box + [NT x 32] W image of the table's
// widest tile, and the ring takes what the staging buffers, barriers, job queue and bias slices leave of the 227 KB
// (less 1 KB for aligning the dynamic shared memory): NT <= 128: 4 x 32 KB, NT = 256: 3 x 48 KB.  The consumers
// hold two slots (the stage being multiplied and the one whose wgmma group has not retired yet), the producer
// fills the rest.
constexpr int MG_RING_BYTES = MG_SMEM_LIMIT - 1024 - MG_OFF_RING;
__host__ __device__ constexpr int mg_slot_bytes(int nt_max) { return MG_A_ATOM + nt_max * 128; }
__host__ __device__ constexpr int mg_slots(int nt_max) {
    return MG_RING_BYTES / mg_slot_bytes(nt_max) < MG_MAX_SLOTS ? MG_RING_BYTES / mg_slot_bytes(nt_max) : MG_MAX_SLOTS;
}
static_assert(mg_slots(256) >= 3, "the widest tile needs a ring of at least three slots");
__host__ __device__ constexpr int mg_k_atoms(int NT) { return NT == 256 ? 1 : 2; }   // per stage of the weight image
constexpr int MG_MAX_LAYERS = 24, MG_MAX_MAPS = 48;
constexpr int MG_BYTES = MG_OFF_RING + MG_RING_BYTES + 1024;
static_assert(MG_BYTES <= MG_SMEM_LIMIT, "exceeds the 227 KB shared-memory limit per CTA");
static_assert(sizeof(fcn_mega_job) == 64 && sizeof(fcn_mega_layer) % 8 == 0, "table record layout");

// Tensor maps and the layer table travel in the kernel parameters (constant bank; CUDA >= 12.1 allows 32 KB).
// With the descriptors in GLOBAL memory every cp.async.bulk.tensor paid an uncached 128-byte descriptor fetch.
struct alignas(64) MegaParams {
    CUtensorMap maps[MG_MAX_MAPS];
    fcn_mega_layer layers[MG_MAX_LAYERS];
    fcn_mega_args a;
    int n_slot, slot_bytes;          // stage ring geometry (mg_slots / mg_slot_bytes of the widest tile)
};
static_assert(sizeof(MegaParams) <= 32000, "kernel parameter space");

__device__ __forceinline__ void mg_tma_load_3d(uint32_t dst, const void *map, int c0, int c1, int c2, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
        "[%0], [%1, {%2, %3, %4}], [%5];\n" ::"r"(dst),
        "l"((uint64_t)map), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
        : "memory");
}
// one staged [32 rows x 32 fp32] box -> the output map (rows past the map are clipped by the TMA unit)
__device__ __forceinline__ void mg_tma_store_3d(const void *map, uint32_t src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4}], [%1];\n" ::"l"(
                     (uint64_t)map),
                 "r"(src), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;\n" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;\n" ::: "memory"); }

__device__ __forceinline__ int ld_acquire_gpu(const int *p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_release_gpu_add(int *p, int v) {
    asm volatile("red.release.gpu.global.add.s32 [%0], %1;\n" ::"l"(p), "r"(v) : "memory");
}
// Between the generic and the async proxy on global memory: on the consumer side, generic-proxy writes of other SMs
// (observed through the acquire above) -> subsequent TMA reads; on the store side, this thread's completed TMA
// stores -> its release of the tile counter.
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;\n" ::: "memory"); }

// Phase timeline (off unless fcn_mega_args.dbg_clocks is set): one row of MG_DBG_ROW clock64 values per job, for
// the first MG_DBG_JOBS jobs of every CTA, at dbg_clocks[(blockIdx.x * MG_DBG_JOBS + q) * MG_DBG_ROW]:
//   [0] TMA lane took the job  [1] job index  [2] scheduler fetched it  [3] its dependencies were met
//   [4] TMA lane issued its last box  [5] TMA clocks spent in `empty` waits
//   [6 + 4 wg] first `full` satisfied  [7 + 4 wg] clocks in `full` waits  [8 + 4 wg] last MMA retired
//   [9 + 4 wg] epilogue done: tile staged, or heads rows decoded (warp 0 of consumer warpgroup wg)
//   [14] layer  [15] SM id
//   store warp: [20] first staged half received  [21] last box store issued  [22] tile counter published
// Clocks are per SM: compare them within a row or a CTA only.
constexpr int MG_DBG_JOBS = 64, MG_DBG_ROW = 32;
__device__ __forceinline__ long long *mg_dbg_row(const fcn_mega_args &p, uint32_t q) {
    return (p.dbg_clocks != nullptr && q < MG_DBG_JOBS)
               ? p.dbg_clocks + MG_DBG_ROW * ((size_t)blockIdx.x * MG_DBG_JOBS + q)
               : nullptr;
}
__device__ __forceinline__ int smid() {
    int v;
    asm volatile("mov.u32 %0, %%smid;\n" : "=r"(v));
    return v;
}

// One job of a consumer warpgroup: the K loop of its 64 rows x NT columns over the stage ring (ring position
// `st`, phase `ph` run on across jobs), then the epilogue.  A stage is handed back when the wgmma group that read
// it has retired.  `stg` is this warpgroup's staging buffer, `nstg` the number of halves it has staged so far
// (the parity of `staged` / `staging_free`), `bias` the job's NT-column bias slice in shared memory.
template <int NT>
__device__ __forceinline__ void mg_job(const MegaParams &P, const fcn_mega_layer &L, int m_tile, int n_tile,
                                       uint32_t &st, uint32_t &ph, uint8_t *ring, uint64_t *full, uint64_t *empty,
                                       uint32_t stg, uint64_t *staged, uint64_t *staging_free, uint32_t &nstg,
                                       const float *bias, int *flags, long long *dbg) {
    const fcn_mega_args &p = P.a;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, wq = warp & 3, t = tid & 127;
    const int NS = L.n_stage * L.k_atoms;                              // 32-wide K stages of this tile
    const uint32_t n_slot = (uint32_t)P.n_slot, slot16 = (uint32_t)P.slot_bytes >> 4;
    const uint64_t adesc0 = make_desc_sw128(smem_u32(ring) + wg * (64 * 128));
    const uint64_t bdesc0 = make_desc_sw128(smem_u32(ring) + MG_A_ATOM);
    float acc[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
    int prev = -1;
    long long t_first = 0, t_full = 0;                                 // timeline (dbg != nullptr only)
    for (int s = 0; s < NS; ++s) {
        const long long t0 = dbg ? clock64() : 0;
        mbar_wait(&full[st], ph);
        if (dbg) {
            const long long t1 = clock64();
            t_full += t1 - t0;
            if (s == 0) t_first = t1;
        }
        const uint64_t ad = adesc0 + (uint64_t)(st * slot16);
        const uint64_t bd = bdesc0 + (uint64_t)(st * slot16);
        wgmma_fence();
        fence_acc(acc);
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_tf32<NT>(acc, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (s | k) != 0);
        wgmma_commit();
        fence_acc(acc);
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = (int)st;
        if (++st == n_slot) { st = 0; ph ^= 1; }
    }
    wgmma_wait<0>();
    fence_acc(acc);
    if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
    if (dbg && lane == 0) { dbg[0] = t_first; dbg[1] = t_full; dbg[2] = clock64(); }

    const int rbase = m_tile * MG_ROWS + 64 * wg;                     // first flattened GEMM row of this warpgroup
    if (!L.is_heads) {
        // +bias (+ReLU, TF32 rounding) -> the staging buffer; the store warp writes it through the output map.
        // One GEMM row holds `up` consecutive output positions (pixel shuffle of the transposed convs): column
        // n = jj*Cout + co -> output position rt*up + jj.  Cout % 32 == 0, so a 32-column box has one jj.  Pad
        // positions (past T_out / T_store) are staged as zeros: the next layer's taps read them.
        // Fragment (row y, columns 2c, 2c+1 of group j) -> box (j / 4, y / 32), row y % 32, 16-byte chunk
        // (2 (j % 4) + c / 2) ^ (y % 8): the eight rows of a warp store land in eight different chunks.
        constexpr int CW = NT < MG_STG_COLS ? NT : MG_STG_COLS;        // columns per staged half
        int rt[2];
#pragma unroll
        for (int half = 0; half < 2; ++half) rt[half] = (rbase + 16 * wq + (lane >> 2) + 8 * half) % L.P_m;
        const uint32_t row_off = (uint32_t)(wq >> 1) * MG_BOX_BYTES + (uint32_t)(16 * (wq & 1) + (lane >> 2)) * 128u;
        const uint32_t sub = (uint32_t)(lane & 1) * 8u;
#pragma unroll
        for (int h = 0; h < NT / CW; ++h) {
            mbar_wait(staging_free, (nstg & 1) ^ 1);                   // the store warp has read the previous half
#pragma unroll
            for (int cb = 0; cb < CW / 32; ++cb) {
                const int jj = (n_tile * NT + h * CW + 32 * cb) / L.Cout;
                bool keep[2];
#pragma unroll
                for (int half = 0; half < 2; ++half)
                    keep[half] = rt[half] < L.T_out && rt[half] * L.up + jj < L.T_store;
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int j = h * (CW / 8) + cb * 4 + u;           // accumulator column group
                    const float2 bb = *(const float2 *)(bias + 8 * j + 2 * (lane & 3));
                    const uint32_t chunk = (uint32_t)((2 * u + ((lane & 3) >> 1)) ^ ((lane >> 2) & 7));
#pragma unroll
                    for (int half = 0; half < 2; ++half) {
                        float2 o = make_float2(0.f, 0.f);
                        if (keep[half]) {
                            o = make_float2(acc[4 * j + 2 * half] + bb.x, acc[4 * j + 2 * half + 1] + bb.y);
                            if (L.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
                            if (L.round_out) { o.x = to_tf32(o.x); o.y = to_tf32(o.y); }
                        }
                        const uint32_t a = stg + (uint32_t)(2 * cb) * MG_BOX_BYTES + row_off + (uint32_t)half * 1024u +
                                           (chunk << 4) + sub;
                        asm volatile("st.shared.v2.f32 [%0], {%1, %2};\n" ::"r"(a), "f"(o.x), "f"(o.y) : "memory");
                    }
                }
            }
            fence_proxy_async();                                       // generic smem writes -> the TMA unit
            __syncwarp();
            if (lane == 0) mbar_arrive(staged);
            ++nstg;
        }
        if (dbg && lane == 0) dbg[3] = clock64();
        return;
    }
    // heads (NT = 64): store the logits rows, then thread t < 64 of the warpgroup decodes row rbase + t into the
    // local block and the peers' gather buffers
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int r = rbase + 16 * wq + (lane >> 2) + 8 * half;
        const int b = r / L.P_m, rt = r - b * L.P_m;
        if (r >= L.n_rows || rt >= L.T_out) continue;
        float *out = L.out + ((size_t)b * L.P_store + rt) * L.ld_out;
#pragma unroll
        for (int j = 0; j < NT / 8; ++j) {
            const int n = n_tile * NT + 8 * j + 2 * (lane & 3);
            if (n >= L.Cout) continue;
            const float2 bb = __ldg((const float2 *)(L.bias + n));
            *(float2 *)(out + n) = make_float2(acc[4 * j + 2 * half] + bb.x, acc[4 * j + 2 * half + 1] + bb.y);
        }
    }
    asm volatile("bar.sync %0, 128;\n" ::"r"(2 + wg) : "memory");   // logits rows of this warpgroup are complete
    {
        const int r = rbase + t;
        const int b = r / L.P_m, rt = r - b * L.P_m;
        if (t < 64 && r < L.n_rows && rt < L.T_out)
            decode_row(L.out + ((size_t)b * L.P_store + rt) * L.ld_out, b * p.T + rt, b, rt, p.T, p.NH, p.NS,
                       p.center_ref, p.mean_size, (const DecodeOut *)p.outs, 1);
    }
    if (p.n_out > 1) {
        // Multi-GPU: replicate this warpgroup's decoded rows into the peers' gather buffers.  The valid rows of a
        // row range are ONE contiguous range of output rows (pad rows have no output row), so each of the six
        // arrays is a contiguous run: copied with consecutive threads -> consecutive floats (full 128-byte NVLink
        // write packets instead of per-row scattered 4-byte remote stores).
        __threadfence();
        asm volatile("bar.sync %0, 128;\n" ::"r"(2 + wg) : "memory");
        const int rfirst = rbase, rlast = min(rfirst + 64, L.n_rows) - 1;
        int b0 = rfirst / L.P_m, t0 = rfirst - b0 * L.P_m;
        if (t0 >= L.T_out) { ++b0; t0 = 0; }
        int b1 = rlast / L.P_m, t1 = rlast - b1 * L.P_m;
        if (t1 >= L.T_out) t1 = L.T_out - 1;
        const int R_lo = b0 * p.T + t0, R_hi = b1 * p.T + t1 + 1;     // [R_lo, R_hi) output rows
        if (rlast >= rfirst && R_hi > R_lo && b0 < p.B) {
            const int widths[6] = {2, 3, 1, 3, p.NH, p.NS};
            const float *const *loc = (const float *const *)&p.outs[0];
#pragma unroll 1
            for (int a6 = 0; a6 < 6; ++a6) {
                const size_t base = (size_t)R_lo * widths[a6];
                const int nflt = (R_hi - R_lo) * widths[a6];
                // four independent loads in flight per thread (the rows were just written: L2 latency),
                // then the posted remote stores
#pragma unroll 1
                for (int i = t; i < nflt; i += 512) {
                    float v[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u)
                        v[u] = (i + 128 * u < nflt) ? __ldcg(loc[a6] + base + i + 128 * u) : 0.f;
                    for (int o = 1; o < p.n_out; ++o) {
                        float *dst = ((float *const *)&p.outs[o])[a6] + base + i;
#pragma unroll
                        for (int u = 0; u < 4; ++u)
                            if (i + 128 * u < nflt) dst[128 * u] = v[u];
                    }
                }
            }
        }
        // no system-scope fence here: nothing consumes a heads tile's counter remotely; every thread fences its
        // remote stores ONCE before the CTA reports completion (end of the kernel), and the last CTA raises the
        // epoch flags after all CTAs have reported
    }
    __threadfence();
    __syncwarp();
    if (lane == 0) red_release_gpu_add(flags + L.flag_base + m_tile, 1);
    if (dbg && lane == 0) dbg[3] = clock64();
}

__global__ void __launch_bounds__(MG_THREADS, 1)
fcn_mega_kernel(const __grid_constant__ MegaParams P) {
    const fcn_mega_args &p = P.a;
    extern __shared__ uint8_t smem_dyn[];
    uint8_t *smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
    uint8_t *ring = smem + MG_OFF_RING;
    const uint32_t stg0 = smem_u32(smem);           // staging buffer of warpgroup wg at stg0 + wg * MG_STG_BYTES
    uint64_t *bars = (uint64_t *)(smem + MG_OFF_BAR);
    uint64_t *full = bars, *empty = bars + MG_MAX_SLOTS;
    uint64_t *job_full = bars + 2 * MG_MAX_SLOTS, *job_empty = job_full + MG_JOBQ, *taken = job_empty + MG_JOBQ;
    uint64_t *staged = taken + 1, *staging_free = staged + 2;
    fcn_mega_job *jobq = (fcn_mega_job *)(smem + MG_OFF_JOBQ);
    float *bias_q = (float *)(smem + MG_OFF_BIAS);  // bias slice of queue entry i at bias_q + MG_BIAS_FLOATS i
    const fcn_mega_layer *s_layers = P.layers;      // kernel parameters (constant bank)

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        for (int i = 0; i < MG_MAX_SLOTS; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], MG_MMA_WARPS); }
        // a queue entry is read by the 8 consumer warps, the TMA lane and the store warp; the consumers release it
        // after their epilogue, which reads the entry's bias slice
        for (int i = 0; i < MG_JOBQ; ++i) { mbar_init(&job_full[i], 1); mbar_init(&job_empty[i], MG_MMA_WARPS + 2); }
        mbar_init(taken, 1);
        for (int i = 0; i < 2; ++i) { mbar_init(&staged[i], 4); mbar_init(&staging_free[i], 1); }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();                 // feature maps come from the PointNet kernels; prologue above overlapped their tail
    pdl_launch_dependents();

    int *job_counter = p.sync, *done_ctas = p.sync + 1, *epoch = p.sync + 2, *flags = p.sync + 4;

    if (warp == MG_SCHED_WARP) {
        // ================= scheduler: fetches job q+1 and waits for its producer tiles while job q streams ========
        // A job enters the queue only once its dependencies are met, so the TMA lane never waits on other CTAs.
        // Job q+1 is taken (atomicAdd) only after the TMA lane has started job q: the CTA holds at most one job that
        // nobody works on yet, and later CTAs find the rest.  Deadlock-free as before: the jobs of a CTA are taken in
        // table order and each waits only on earlier jobs, which are running or done.
        for (uint32_t q = 0;; ++q) {
            if (q > 0) mbar_wait(taken, (q - 1) & 1);
            int j = 0;
            if (lane == 0) j = atomicAdd(job_counter, 1);
            j = __shfl_sync(0xffffffffu, j, 0);
            long long *dbg = mg_dbg_row(p, q);
            if (dbg && lane == 0) { dbg[1] = j; dbg[2] = clock64(); }
            const uint32_t slot = q % MG_JOBQ;
            mbar_wait(&job_empty[slot], ((q / MG_JOBQ) & 1) ^ 1);
            int4 *dst = (int4 *)&jobq[slot];
            if (j < p.n_jobs) {
                if (lane < 4) dst[lane] = __ldg((const int4 *)(p.jobs + j) + lane);
            } else if (lane == 0) {
                dst[0] = make_int4(-1, 0, 0, 0);
            }
            __syncwarp();
            if (j < p.n_jobs) {
                // all counters of the producer tiles at once: lane i polls counters i, i+32, ... of each dependency
                const fcn_mega_job &job = jobq[slot];
                uint32_t spins = 0;
                bool ready;
                do {
                    ready = true;
                    for (int d = 0; d < job.n_dep; ++d)
                        for (int i = lane; i < job.dep[d].count; i += 32)
                            if (ld_acquire_gpu(flags + job.dep[d].first + i) < job.dep[d].target) ready = false;
                    if (++spins > (1u << 24)) __trap();   // protocol bug -> launch failure, not a hang
                } while (!__all_sync(0xffffffffu, ready));
            }
            if (dbg && lane == 0) dbg[3] = clock64();
            __syncwarp();
            if (lane == 0) mbar_arrive(&job_full[slot]);     // release: descriptor + the acquired counters
            if (j >= p.n_jobs) break;
        }
    } else if (warp == MG_TMA_WARP) {
        // ================= TMA producer (one lane): waits only on the ring and the job queue =================
        if (lane == 0) {
            const uint32_t n_slot = (uint32_t)P.n_slot, slot_bytes = (uint32_t)P.slot_bytes;
            uint32_t st = 0, ph = 0;                 // ring position and phase, running across jobs
            for (uint32_t q = 0;; ++q) {
                const uint32_t slot = q % MG_JOBQ;
                mbar_wait(&job_full[slot], (q / MG_JOBQ) & 1);
                const int layer = jobq[slot].layer, m_tile = jobq[slot].m_tile, n_tile = jobq[slot].n_tile;
                const int n_dep = jobq[slot].n_dep;
                mbar_arrive(&job_empty[slot]);
                mbar_arrive(taken);                  // the scheduler may fetch the next job
                if (layer < 0) break;
                long long *dbg = mg_dbg_row(p, q);
                long long t_empty = 0;
                if (dbg) { dbg[0] = clock64(); dbg[14] = layer; dbg[15] = smid(); }
                const fcn_mega_layer &L = s_layers[layer];
                const int r0 = m_tile * MG_ROWS;
                const int NS = L.n_stage * L.k_atoms;
                const uint32_t w_bytes = (uint32_t)(L.NT * 128);          // one [NT rows x 32 tf32] atom
                const uint8_t *wsrc = (const uint8_t *)L.w_tc + (size_t)n_tile * NS * w_bytes;
                // the scheduler acquired the producer tiles' counters (generic proxy): order them before the TMA reads
                if (n_dep > 0) fence_proxy_async_global();
                int seg = 0, kbi = 0;                 // running (segment, 32-channel block inside the segment)
                for (int s = 0; s < NS; ++s) {
                    const long long t0 = dbg ? clock64() : 0;
                    mbar_wait(&empty[st], ph ^ 1);
                    if (dbg) t_empty += clock64() - t0;
                    uint8_t *sl = ring + st * slot_bytes;
                    // the job's bias slice rides on its first stage (the consumers read it in the epilogue)
                    const bool with_bias = s == 0 && !L.is_heads;
                    mbar_arrive_expect_tx(&full[st], MG_A_ATOM + w_bytes + (with_bias ? L.NT * 4 : 0));
                    if (with_bias) bulk_g2s(bias_q + MG_BIAS_FLOATS * slot, L.bias + n_tile * L.NT, L.NT * 4, &full[st]);
                    bulk_g2s(sl + MG_A_ATOM, wsrc + (size_t)s * w_bytes, w_bytes, &full[st]);
                    if (seg < L.n_seg) {
                        const fcn_mega_seg &sgm = L.seg[seg];
                        mg_tma_load_3d(smem_u32(sl), &P.maps[sgm.map_idx], kbi * 32, r0 * sgm.stride + sgm.tap, 0, &full[st]);
                        if (++kbi >= sgm.kblocks) { kbi = 0; ++seg; }
                    } else {   // K padding block: a box fully outside the channel range -> zeros
                        mg_tma_load_3d(smem_u32(sl), &P.maps[L.seg[0].map_idx], 1 << 20, 0, 0, &full[st]);
                    }
                    if (++st == n_slot) { st = 0; ph ^= 1; }
                }
                if (dbg) { dbg[4] = clock64(); dbg[5] = t_empty; }
            }
        }
    } else if (warp == MG_STORE_WARP) {
        // ================= store warp (one lane): staged tiles -> TMA stores -> tile counter =================
        // Waits only on the job queue (an entry is full before the consumers start that job), on this CTA's
        // consumers (`staged`) and on its own bulk groups.
        if (lane == 0) {
            uint32_t nstg[2] = {0, 0};               // halves received per warpgroup (parity of `staged`)
            for (uint32_t q = 0;; ++q) {
                const uint32_t slot = q % MG_JOBQ;
                mbar_wait(&job_full[slot], (q / MG_JOBQ) & 1);
                const int layer = jobq[slot].layer, m_tile = jobq[slot].m_tile, n_tile = jobq[slot].n_tile;
                mbar_arrive(&job_empty[slot]);
                if (layer < 0) break;
                const fcn_mega_layer &L = s_layers[layer];
                if (L.is_heads) continue;            // the heads epilogue stores and publishes by itself
                long long *dbg = mg_dbg_row(p, q);
                const void *map = &P.maps[L.out_map];
                const int cw = L.NT < MG_STG_COLS ? L.NT : MG_STG_COLS, ncols = L.up * L.Cout;
                for (int h = 0; h < L.NT / cw; ++h) {
                    for (int wg = 0; wg < 2; ++wg) {
                        mbar_wait(&staged[wg], nstg[wg]++ & 1);
                        if (dbg && h == 0 && wg == 0) dbg[20] = clock64();
                        const int row0 = m_tile * MG_ROWS + 64 * wg;
                        const uint32_t src = stg0 + (uint32_t)wg * MG_STG_BYTES;
                        for (int cb = 0; cb < cw / 32; ++cb) {
                            const int n0 = n_tile * L.NT + h * cw + 32 * cb;   // columns past up*Cout: padding
                            if (n0 >= ncols) break;
                            const int jj = n0 / L.Cout, c = jj * L.ld_out + L.c_off + (n0 - jj * L.Cout);
                            for (int rb = 0; rb < 2; ++rb)
                                if (row0 + 32 * rb < L.n_rows)
                                    mg_tma_store_3d(map, src + (uint32_t)(2 * cb + rb) * MG_BOX_BYTES, c, row0 + 32 * rb, 0);
                        }
                        bulk_commit();
                        bulk_wait_read_all();        // the TMA unit has read the buffer: the warpgroup may refill it
                        mbar_arrive(&staging_free[wg]);
                    }
                }
                if (dbg) dbg[21] = clock64();
                // the tile's stores are complete; async-proxy writes -> generic release -> the dependent tiles'
                // acquire + fence.proxy.async.global before their TMA loads
                bulk_wait_all();
                fence_proxy_async_global();
                red_release_gpu_add(flags + L.flag_base + m_tile, 1);
                if (dbg) dbg[22] = clock64();
            }
        }
    } else {
        // ================= consumer warpgroups: MMA + epilogue staging of every job, 64 rows each ===========
        const int wg = warp >> 2;
        uint32_t st = 0, ph = 0, nstg = 0;
        const uint32_t stg = stg0 + (uint32_t)wg * MG_STG_BYTES;
        for (uint32_t q = 0;; ++q) {
            const uint32_t slot = q % MG_JOBQ;
            mbar_wait(&job_full[slot], (q / MG_JOBQ) & 1);
            const int layer = jobq[slot].layer, m_tile = jobq[slot].m_tile, n_tile = jobq[slot].n_tile;
            if (layer < 0) break;
            const fcn_mega_layer &L = s_layers[layer];
            long long *dbg = (warp & 3) == 0 ? mg_dbg_row(p, q) : nullptr;   // warp 0 of each warpgroup
            if (dbg) dbg += 6 + 4 * wg;
            const float *bias = bias_q + MG_BIAS_FLOATS * slot;
            if (L.NT == 256)
                mg_job<256>(P, L, m_tile, n_tile, st, ph, ring, full, empty, stg, &staged[wg], &staging_free[wg], nstg,
                            bias, flags, dbg);
            else if (L.NT == 128)
                mg_job<128>(P, L, m_tile, n_tile, st, ph, ring, full, empty, stg, &staged[wg], &staging_free[wg], nstg,
                            bias, flags, dbg);
            else
                mg_job<64>(P, L, m_tile, n_tile, st, ph, ring, full, empty, stg, &staged[wg], &staging_free[wg], nstg,
                           bias, flags, dbg);
            __syncwarp();
            if (lane == 0) mbar_arrive(&job_empty[slot]);   // descriptor and bias slice no longer needed
        }
    }
    if (p.n_out > 1) __threadfence_system();      // this thread's remote (NVLink) result stores, if any
    __syncthreads();
    // self-cleaning: the last CTA out resets the scheduler state for the next forward and, on the multi-GPU
    // path, raises this rank's epoch flag in every peer (all result rows were fenced at system scope above)
    int &s_last = *(int *)(bars + MG_NBAR);         // behind the barriers: no static shared memory
    if (tid == 0) {
        __threadfence();
        s_last = atomicAdd(done_ctas, 1) == (int)gridDim.x - 1;
    }
    __syncthreads();
    if (s_last) {
        __threadfence();
        for (int i = tid; i < p.n_flags; i += MG_THREADS) flags[i] = 0;
        __syncthreads();
        if (tid == 0) {
            *job_counter = 0;
            *done_ctas = 0;
            const int e = *epoch + 1;
            *epoch = e;
            __threadfence_system();
            for (int o = 0; o < p.n_flag_out; ++o)
                if (p.flag_out[o] != nullptr) *(volatile int *)p.flag_out[o] = e;
            __threadfence_system();
        }
    }
}

}  // namespace fcn

using namespace fcn;

extern "C" int fcn_mega_forward(const fcn_mega_args *args, fcn_stream_t stream) {
    FCN_REQUIRE(args != nullptr, "args is NULL");
    const fcn_mega_args &a = *args;
    FCN_REQUIRE(a.n_jobs >= 0 && a.n_layers >= 1 && a.n_flags >= 0, "bad table sizes");
    FCN_REQUIRE(a.layers && a.jobs && a.tmaps && a.sync, "NULL table pointer");
    FCN_REQUIRE(a.n_layers <= MG_MAX_LAYERS && a.n_maps >= 1 && a.n_maps <= MG_MAX_MAPS, "too many layers / tensor maps");
    FCN_REQUIRE(a.n_out >= 0 && a.n_out <= FCN_MAX_PEERS && a.n_flag_out >= 0 && a.n_flag_out <= FCN_MAX_PEERS,
                "too many output sets");
    FCN_REQUIRE(a.NH >= 1 && a.NH <= DEC_MAX_BINS && a.NS >= 1 && a.NS <= DEC_MAX_BINS, "bad decode sizes");
    int nt_max = 0;
    for (int i = 0; i < a.n_layers; ++i) {
        const fcn_mega_layer &L = a.layers[i];
        FCN_REQUIRE((L.NT == 64 || L.NT == 128 || L.NT == 256) && L.k_atoms == mg_k_atoms(L.NT),
                    "layer tile width must be 64, 128 or 256, with k_atoms = 1 for 256 and 2 otherwise");
        FCN_REQUIRE(L.is_heads || ((uintptr_t)L.bias & 15) == 0,
                    "layer bias must be 16-byte aligned (its NT-column slices are bulk-copied)");
        // every heads job decodes whole logit rows right after storing its own NT columns
        FCN_REQUIRE(!L.is_heads || L.n_tiles_n == 1, "the heads layer must be a single N tile (ld_logit <= 128)");
        nt_max = L.NT > nt_max ? L.NT : nt_max;
    }
    if (a.n_jobs == 0) return FCN_OK;
    static_assert(sizeof(DecodeOut) == sizeof(fcn_decode_out), "decode output block layout");
    int grid = a.grid > 0 ? a.grid : sm_count();
    if (grid > a.n_jobs) grid = a.n_jobs;
    if (grid > sm_count()) grid = sm_count();
    FCN_CUDA(cudaFuncSetAttribute(fcn_mega_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MG_BYTES));
    MegaParams P;
    memcpy(P.maps, a.tmaps, sizeof(CUtensorMap) * a.n_maps);   // HOST arrays -> kernel parameters
    memcpy(P.layers, a.layers, sizeof(fcn_mega_layer) * a.n_layers);
    P.a = a;
    P.n_slot = mg_slots(nt_max);              // every accepted tile width fits (static_assert on mg_slots(256))
    P.slot_bytes = mg_slot_bytes(nt_max);
    static const int prio = env_priority("FCN_PRIO_CONV");
    FCN_CUDA(launch_pdl_prio(prio, fcn_mega_kernel, dim3(grid), dim3(MG_THREADS), (size_t)MG_BYTES, (cudaStream_t)stream, P));
    return FCN_OK;
}
