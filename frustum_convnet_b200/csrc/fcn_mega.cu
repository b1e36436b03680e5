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
//   * layer-to-layer dependencies are per row tile: the epilogue of a tile publishes a counter
//     (release, gpu scope); the TMA producer of a consumer tile acquires the counters of the (<= 4) source
//     tiles it reads (taps +-1, stride 2, pixel-shuffled transposed convs), then crosses to the async proxy;
//   * inside a CTA the same warp-specialised pipeline as conv_gemm_tma.cu, made continuous across jobs: warp 8 =
//     scheduler + TMA producer (A boxes by cp.async.bulk.tensor with the conv taps / stride in the coordinates,
//     weight stage images by bulk copies), warps 0-7 = two consumer warpgroups (wgmma, 64 rows each, N = NT =
//     256 | 128 | 64) that also run the epilogue; the smem stage ring runs across job boundaries (the next job's
//     operands stream while the current one is still multiplied or stored);
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
constexpr int MG_MMA_WARPS = 8;      // warps 0-7: two consumer warpgroups (MMA + epilogue); warp 8: scheduler + TMA
constexpr int MG_THREADS = (MG_MMA_WARPS + 1) * 32;
constexpr int MG_NSTAGE = 3;         // stage slot: 2 x 16 KB of A + 32 KB of W (NT <= 128: 64-wide K; NT = 256: 32-wide)
constexpr int MG_A_ATOM = MG_ROWS * 128, MG_A_STAGE = 2 * MG_A_ATOM;
constexpr int MG_W_STAGE = 2 * 128 * 128;                     // two [128 x 32] atoms or one [256 x 32] atom
__host__ __device__ constexpr int mg_k_atoms(int NT) { return NT == 256 ? 1 : 2; }   // 32-wide K atoms per stage
constexpr int MG_OFF_W = MG_NSTAGE * MG_A_STAGE;
constexpr int MG_OFF_BAR = MG_OFF_W + MG_NSTAGE * MG_W_STAGE;
constexpr int MG_JOBQ = 4;                                    // job descriptors in flight inside a CTA
constexpr int MG_NBAR = 2 * MG_NSTAGE + 2 * MG_JOBQ;          // full/empty, job_full/job_empty
constexpr int MG_OFF_JOBQ = MG_OFF_BAR + MG_NBAR * 8;         // fcn_mega_job[MG_JOBQ] (64 B each)
constexpr int MG_MAX_LAYERS = 24, MG_MAX_MAPS = 48;
constexpr int MG_BYTES = MG_OFF_JOBQ + MG_JOBQ * (int)sizeof(fcn_mega_job) + 1024;
static_assert(MG_BYTES <= 232448, "exceeds the 227 KB shared-memory limit per CTA");
static_assert(sizeof(fcn_mega_job) == 64 && sizeof(fcn_mega_layer) % 8 == 0, "table record layout");

// Tensor maps and the layer table travel in the kernel parameters (constant bank; CUDA >= 12.1 allows 32 KB).
// With the descriptors in GLOBAL memory every cp.async.bulk.tensor paid an uncached 128-byte descriptor fetch.
struct alignas(64) MegaParams {
    CUtensorMap maps[MG_MAX_MAPS];
    fcn_mega_layer layers[MG_MAX_LAYERS];
    fcn_mega_args a;
};
static_assert(sizeof(MegaParams) <= 32000, "kernel parameter space");

__device__ __forceinline__ void mg_tma_load_3d(uint32_t dst, const void *map, int c0, int c1, int c2, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
        "[%0], [%1, {%2, %3, %4}], [%5];\n" ::"r"(dst),
        "l"((uint64_t)map), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
        : "memory");
}

__device__ __forceinline__ int ld_acquire_gpu(const int *p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_release_gpu_add(int *p, int v) {
    asm volatile("red.release.gpu.global.add.s32 [%0], %1;\n" ::"l"(p), "r"(v) : "memory");
}
// generic-proxy writes of other SMs (observed through the acquire above) -> subsequent async-proxy (TMA) reads
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;\n" ::: "memory"); }

// One job of a consumer warpgroup: the K loop of its 64 rows x NT columns over the stage ring (`stage` runs on
// across jobs), then the epilogue.  A stage is handed back when the wgmma group that read it has retired.
template <int NT>
__device__ __forceinline__ void mg_job(const MegaParams &P, const fcn_mega_layer &L, int m_tile, int n_tile,
                                       uint32_t &stage, uint8_t *sA, uint8_t *sW, uint64_t *full, uint64_t *empty,
                                       int *flags) {
    const fcn_mega_args &p = P.a;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, wq = warp & 3, t = tid & 127;
    // 32-wide K atoms per stage (the layer table's k_atoms, checked on the host): a compile-time count keeps every
    // wgmma of a stage in straight-line code
    constexpr int KA = mg_k_atoms(NT);
    const int NS = L.n_stage;
    const uint32_t w_atom16 = (uint32_t)(NT * 128) >> 4;              // second 32-wide K atom of a W stage
    const uint64_t adesc0 = make_desc_sw128(smem_u32(sA) + wg * (64 * 128));
    const uint64_t bdesc0 = make_desc_sw128(smem_u32(sW));
    float acc[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int s = 0; s < NS; ++s, ++stage) {
        const uint32_t st = stage % MG_NSTAGE, ph = (stage / MG_NSTAGE) & 1;
        mbar_wait(&full[st], ph);
        const uint64_t ad = adesc0 + (uint64_t)(st * (MG_A_STAGE >> 4));
        const uint64_t bd = bdesc0 + (uint64_t)(st * (MG_W_STAGE >> 4));
        wgmma_fence();
        fence_acc(acc);
#pragma unroll
        for (int a = 0; a < KA; ++a)
#pragma unroll
            for (int k = 0; k < 4; ++k)
                wgmma_tf32<NT>(acc, ad + (uint64_t)(a * (MG_A_ATOM >> 4) + 2 * k), bd + (uint64_t)(a * w_atom16 + 2 * k),
                               (s | a | k) != 0);
        wgmma_commit();
        fence_acc(acc);
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = (int)st;
    }
    wgmma_wait<0>();
    fence_acc(acc);
    if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);

    const int rbase = m_tile * MG_ROWS + 64 * wg;                     // first flattened GEMM row of this warpgroup
    if (!L.is_heads) {
        // +bias (+ReLU, TF32 rounding) -> the output map.  One GEMM row holds `up` consecutive output positions
        // (pixel shuffle of the transposed convs): row r, column n = jj*Cout + co -> out[r][jj][c_off + co].
        // Pad positions (past T_out / T_store) are written as zeros: the next layer's taps read them.
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int r = rbase + 16 * wq + (lane >> 2) + 8 * half;
            if (r >= L.n_rows) continue;
            const int rt = r % L.P_m;
            float *orow = L.out + (size_t)r * L.up * L.ld_out + L.c_off;
#pragma unroll
            for (int j = 0; j < NT / 8; ++j) {
                const int n = n_tile * NT + 8 * j + 2 * (lane & 3);   // even; the pair never crosses a Cout boundary
                if (n >= L.up * L.Cout) continue;
                const int jj = n / L.Cout, co = n - jj * L.Cout;
                float2 o = make_float2(0.f, 0.f);
                if (rt < L.T_out && rt * L.up + jj < L.T_store) {
                    const float2 bb = __ldg((const float2 *)(L.bias + n));
                    o = make_float2(acc[4 * j + 2 * half] + bb.x, acc[4 * j + 2 * half + 1] + bb.y);
                    if (L.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
                    if (L.round_out) { o.x = to_tf32(o.x); o.y = to_tf32(o.y); }
                }
                *(float2 *)(orow + jj * L.ld_out + co) = o;
            }
        }
        // publish: one count per consumer warp once its stores are visible at gpu scope
        __threadfence();
        __syncwarp();
        if (lane == 0) red_release_gpu_add(flags + L.flag_base + m_tile, 1);
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
}

__global__ void __launch_bounds__(MG_THREADS, 1)
fcn_mega_kernel(const __grid_constant__ MegaParams P) {
    const fcn_mega_args &p = P.a;
    extern __shared__ uint8_t smem_dyn[];
    uint8_t *smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
    uint8_t *sA = smem, *sW = smem + MG_OFF_W;
    uint64_t *bars = (uint64_t *)(smem + MG_OFF_BAR);
    uint64_t *full = bars, *empty = bars + MG_NSTAGE;
    uint64_t *job_full = bars + 2 * MG_NSTAGE, *job_empty = job_full + MG_JOBQ;
    fcn_mega_job *jobq = (fcn_mega_job *)(smem + MG_OFF_JOBQ);
    const fcn_mega_layer *s_layers = P.layers;      // kernel parameters (constant bank)

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        for (int i = 0; i < MG_NSTAGE; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], MG_MMA_WARPS); }
        for (int i = 0; i < MG_JOBQ; ++i) { mbar_init(&job_full[i], 1); mbar_init(&job_empty[i], MG_MMA_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();                 // feature maps come from the PointNet kernels; prologue above overlapped their tail
    pdl_launch_dependents();

    int *job_counter = p.sync, *done_ctas = p.sync + 1, *epoch = p.sync + 2, *flags = p.sync + 4;

    if (warp == MG_MMA_WARPS) {
        // ================= scheduler + TMA producer (one lane) =================
        if (lane == 0) {
            uint32_t stage = 0;                       // running K-stage counter across jobs
            // The job index comes from ONE atomicAdd; index and descriptor of job q+1 are fetched while the first
            // K stages of job q are in flight (the fetch chain is two dependent L2 round trips, ~1.8 k clk: issued
            // at the top of a job it left the tensor pipe idle between jobs).
            auto publish = [&](uint32_t q, int j) -> int {     // descriptor -> queue slot q; returns the layer (-1: end)
                const uint32_t slot = q % MG_JOBQ;
                mbar_wait(&job_empty[slot], ((q / MG_JOBQ) & 1) ^ 1);
                int4 *dst = (int4 *)&jobq[slot];
                int layer = -1;
                if (j < p.n_jobs) {
                    const int4 *src = (const int4 *)(p.jobs + j);
                    const int4 a0 = __ldg(src), a1 = __ldg(src + 1), a2 = __ldg(src + 2), a3 = __ldg(src + 3);
                    dst[0] = a0; dst[1] = a1; dst[2] = a2; dst[3] = a3;
                    layer = a0.x;
                } else {
                    dst[0] = make_int4(-1, 0, 0, 0);
                }
                mbar_arrive(&job_full[slot]);         // release: the queue entry is visible to the waiters
                return layer;
            };
            int jcur = atomicAdd(job_counter, 1);
            int layer = publish(0, jcur);
            for (uint32_t q = 0; layer >= 0; ++q) {
                const fcn_mega_job &job = jobq[q % MG_JOBQ];   // own copy in shared memory (slot is reused only
                                                               // after MG_JOBQ more jobs were published)
                const fcn_mega_layer &L = s_layers[layer];
                long long *dbg = (p.dbg_clocks != nullptr && blockIdx.x == 0 && q < 64) ? p.dbg_clocks + 16 * q : nullptr;
                if (dbg) { dbg[0] = clock64(); dbg[1] = jcur; }
                const int r0 = job.m_tile * MG_ROWS;
                const int NS = L.n_stage;
                const int ka = mg_k_atoms(L.NT);
                const uint32_t w_bytes = (uint32_t)(L.NT * 128 * ka);    // [NT rows x 32 tf32] per atom
                const uint32_t a_bytes = (uint32_t)(ka * MG_A_ATOM);
                const uint8_t *wsrc = (const uint8_t *)L.w_tc + (size_t)job.n_tile * NS * w_bytes;
                // weights do not depend on other tiles: the first ring-full of weight stages streams WHILE this
                // tile's dependencies are awaited (only the A boxes wait for the producer tiles).  (Issuing every
                // stage's A boxes individually behind a non-blocking dependency probe is not done.)
                const int npre = NS < MG_NSTAGE ? NS : MG_NSTAGE;
                for (int s = 0; s < npre; ++s) {
                    const uint32_t sg = stage + s, st = sg % MG_NSTAGE, ph = (sg / MG_NSTAGE) & 1;
                    mbar_wait(&empty[st], ph ^ 1);
                    mbar_arrive_expect_tx(&full[st], a_bytes + w_bytes);
                    bulk_g2s(sW + st * MG_W_STAGE, wsrc + (size_t)s * w_bytes, w_bytes, &full[st]);
                }
                const int jnext = atomicAdd(job_counter, 1);   // in flight during the dependency wait below
                // dependencies: the row tiles of the producing layers this tile reads
                const int n_dep = job.n_dep;
                for (int d = 0; d < n_dep; ++d) {
                    const int first = job.dep[d].first, cnt = job.dep[d].count, target = job.dep[d].target;
                    for (int i = 0; i < cnt; ++i) {
                        uint32_t spins = 0;
                        while (ld_acquire_gpu(flags + first + i) < target) {
                            if (++spins > (1u << 24)) __trap();   // protocol bug -> launch failure, not a hang
                        }
                    }
                }
                if (dbg) dbg[2] = clock64();
                if (n_dep > 0) fence_proxy_async_global();
                if (dbg) dbg[3] = clock64();
                int seg = 0, kbi = 0;                 // running (segment, 32-channel block inside the segment)
                int next_layer = -1;
                for (int s = 0; s < NS; ++s, ++stage) {
                    const uint32_t st = stage % MG_NSTAGE, ph = (stage / MG_NSTAGE) & 1;
                    if (s == npre) next_layer = publish(q + 1, jnext);   // first ring-full issued: fetch the next job
                    if (s >= npre) {
                        mbar_wait(&empty[st], ph ^ 1);
                        mbar_arrive_expect_tx(&full[st], a_bytes + w_bytes);
                        bulk_g2s(sW + st * MG_W_STAGE, wsrc + (size_t)s * w_bytes, w_bytes, &full[st]);
                    }
                    for (int a = 0; a < ka; ++a) {
                        const uint32_t dst = smem_u32(sA) + st * MG_A_STAGE + a * MG_A_ATOM;
                        if (seg < L.n_seg) {
                            const fcn_mega_seg &sgm = L.seg[seg];
                            mg_tma_load_3d(dst, &P.maps[sgm.map_idx], kbi * 32, r0 * sgm.stride + sgm.tap, 0, &full[st]);
                            if (++kbi >= sgm.kblocks) { kbi = 0; ++seg; }
                        } else {   // K padding block: a box fully outside the channel range -> zeros
                            mg_tma_load_3d(dst, &P.maps[L.seg[0].map_idx], 1 << 20, 0, 0, &full[st]);
                        }
                    }
                }
                if (NS <= npre) next_layer = publish(q + 1, jnext);
                if (dbg) dbg[4] = clock64();
                layer = next_layer;
                jcur = jnext;
            }
        }
    } else {
        // ================= consumer warpgroups: MMA + epilogue of every job, 64 rows each =================
        uint32_t stage = 0;
        for (uint32_t q = 0;; ++q) {
            const uint32_t slot = q % MG_JOBQ;
            mbar_wait(&job_full[slot], (q / MG_JOBQ) & 1);
            const int layer = jobq[slot].layer, m_tile = jobq[slot].m_tile, n_tile = jobq[slot].n_tile;
            __syncwarp();
            if (lane == 0) mbar_arrive(&job_empty[slot]);
            if (layer < 0) break;
            const fcn_mega_layer &L = s_layers[layer];
            if (L.NT == 256) mg_job<256>(P, L, m_tile, n_tile, stage, sA, sW, full, empty, flags);
            else if (L.NT == 128) mg_job<128>(P, L, m_tile, n_tile, stage, sA, sW, full, empty, flags);
            else mg_job<64>(P, L, m_tile, n_tile, stage, sA, sW, full, empty, flags);
        }
    }
    if (p.n_out > 1) __threadfence_system();      // this thread's remote (NVLink) result stores, if any
    __syncthreads();
    // self-cleaning: the last CTA out resets the scheduler state for the next forward and, on the multi-GPU
    // path, raises this rank's epoch flag in every peer (all result rows were fenced at system scope above)
    __shared__ int s_last;
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
    for (int i = 0; i < a.n_layers; ++i) {
        const fcn_mega_layer &L = a.layers[i];
        FCN_REQUIRE((L.NT == 64 || L.NT == 128 || L.NT == 256) && L.k_atoms == mg_k_atoms(L.NT),
                    "layer tile width must be 64, 128 or 256, with k_atoms = 1 for 256 and 2 otherwise");
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
    static const int prio = env_priority("FCN_PRIO_CONV");
    FCN_CUDA(launch_pdl_prio(prio, fcn_mega_kernel, dim3(grid), dim3(MG_THREADS), (size_t)MG_BYTES, (cudaStream_t)stream, P));
    return FCN_OK;
}
