// fcn_sunrgbd_depth_cloud (C ABI section (24)): SUN-RGBD depth images to section (23)'s (F, P, 6) clouds, the
// reference's read_3d_points (sunrgbd/read_3d_points.py) per pixel with an order-preserving compaction of the valid
// pixels.  Tile t of frame f is pixels [t * SD_TILE, (t + 1) * SD_TILE) of the H x W grid in row-major order; the
// frame's h x w crop is a subset of that grid in the same order, so the crop's row-major rank of a valid pixel is
// its rank among the grid's valid pixels.  In order:
//   sd_count   per (tile, frame): the tile's valid pixels;
//   sd_scan    one CTA per frame: an exclusive scan of its tile counts in place, the frame's count and status bits;
//   sd_write   per (tile, frame): the same traversal ranks each valid pixel (warp ballots in scan order) and writes
//              its point at the tile's first rank plus its rank; a tile that starts at or past P writes nothing.
#include <cub/block/block_scan.cuh>

#include "common.cuh"
#include "input_builder.cuh"

namespace fcn {

constexpr int SD_THREADS = 256;
constexpr int SD_ITEMS = 8;                         // pixels per thread of a tile
constexpr int SD_TILE = SD_THREADS * SD_ITEMS;
constexpr int SD_WARPS = SD_THREADS / 32;

struct SdWs {
    int32_t *tiles;             // (F, C) per-tile valid pixels, then each tile's first rank
    int32_t *total;             // (F) valid pixels of each frame
};

// frame f's crop, clamped to the capacity
__device__ __forceinline__ void sd_crop(const fcn_sunrgbd_depth_args &a, int f, int &h, int &w) {
    h = min(max(a.image_hw[2 * f], 0), a.height);
    w = min(max(a.image_hw[2 * f + 1], 0), a.width);
}

// pixel g of frame f's grid: its raw depth when it lies in the crop, else 0 (invalid)
__device__ __forceinline__ unsigned sd_raw(const fcn_sunrgbd_depth_args &a, int f, int g, int HW, int h, int w,
                                           int &v, int &u) {
    v = g / a.width;
    u = g - v * a.width;
    if (g >= HW || v >= h || u >= w) return 0u;
    return a.depth[(size_t)f * HW + g];
}

// grid (C, F)
__global__ void __launch_bounds__(SD_THREADS) sd_count_kernel(const fcn_sunrgbd_depth_args a, SdWs s, int C) {
    __shared__ int cnt;
    const int f = blockIdx.y, HW = a.height * a.width, g0 = blockIdx.x * SD_TILE;
    int h, w;
    sd_crop(a, f, h, w);
    if (threadIdx.x == 0) cnt = 0;
    int n = 0;
#pragma unroll
    for (int q = 0; q < SD_ITEMS; ++q) {
        int v, u;
        n += sd_raw(a, f, g0 + q * SD_THREADS + threadIdx.x, HW, h, w, v, u) != 0u;
    }
    n = __reduce_add_sync(0xffffffffu, n);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) atomicAdd(&cnt, n);
    __syncthreads();
    if (threadIdx.x == 0) s.tiles[(size_t)f * C + blockIdx.x] = cnt;
}

// one CTA per frame
__global__ void __launch_bounds__(SD_THREADS) sd_scan_kernel(const fcn_sunrgbd_depth_args a, SdWs s, int C) {
    using Scan = cub::BlockScan<int, SD_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    const int f = blockIdx.x;
    int32_t *t = s.tiles + (size_t)f * C;
    int run = 0;
    for (int c0 = 0; c0 < C; c0 += SD_THREADS) {
        const int c = c0 + threadIdx.x;
        const int v = c < C ? t[c] : 0;
        int x, total;
        Scan(tmp).ExclusiveSum(v, x, total);
        if (c < C) t[c] = run + x;
        run += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const int P = a.point_capacity, h = a.image_hw[2 * f], w = a.image_hw[2 * f + 1];
        s.total[f] = run;
        a.counts[f] = run < P ? run : P;
        const int bits = (run > P ? FCN_FRAME_SCAN_POINTS : 0) | (h > a.height || w > a.width ? FCN_FRAME_PIXELS : 0);
        if (bits) atomicOr(a.status, bits);
    }
}

// grid (C, F).  Round q visits pixels g0 + q * SD_THREADS + threadIdx.x, so rounds, warps and lanes go in scan order:
// a valid pixel's rank is the tile's first rank, the valid pixels of earlier rounds (run), of earlier warps of its
// round (wcnt, double-buffered so one barrier a round suffices) and of earlier lanes of its warp (ballot).
__global__ void __launch_bounds__(SD_THREADS) sd_write_kernel(const fcn_sunrgbd_depth_args a, SdWs s, int C) {
    __shared__ double m[18];
    __shared__ int wcnt[2][SD_WARPS];
    const int f = blockIdx.y, P = a.point_capacity, HW = a.height * a.width, g0 = blockIdx.x * SD_TILE;
    int run = s.tiles[(size_t)f * C + blockIdx.x];
    if (run >= P) return;
    if (threadIdx.x < 18) m[threadIdx.x] = a.calibs[18 * (size_t)f + threadIdx.x];
    int h, w;
    sd_crop(a, f, h, w);
    const bool single = s.total[f] == 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned lt = (1u << lane) - 1u;
    __syncthreads();
    const double *R = m, cx = m[9 + 2], cy = m[9 + 5], fx = m[9 + 0], fy = m[9 + 4];
    for (int q = 0; q < SD_ITEMS && run < P; ++q) {
        int v, u;
        const unsigned raw = sd_raw(a, f, g0 + q * SD_THREADS + threadIdx.x, HW, h, w, v, u);
        const unsigned b = __ballot_sync(0xffffffffu, raw != 0u);
        if (lane == 0) wcnt[q & 1][warp] = __popc(b);
        __syncthreads();
        int r = run + __popc(b & lt), n = 0;
#pragma unroll
        for (int x = 0; x < SD_WARPS; ++x) {
            const int c = wcnt[q & 1][x];
            r += x < warp ? c : 0;
            n += c;
        }
        run += n;
        if (raw == 0u || r >= P) continue;
        const unsigned rot = ((raw >> 3) | (raw << 13)) & 0xffffu;
        float d = __fdiv_rn((float)rot, 1000.f);
        if (d > 8.f) d = 8.f;
        const double z = (double)d;
        const double x3 = __ddiv_rn(__dmul_rn(__dsub_rn((double)u, cx), z), fx);
        const double y3 = __ddiv_rn(__dmul_rn(__dsub_rn((double)v, cy), z), fy);
        float *o = a.clouds + 6 * ((size_t)f * P + r);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const double *Rk = R + 3 * k;
            const double y = single ? __fma_rn(Rk[2], -y3, __fma_rn(Rk[0], x3, __dmul_rn(Rk[1], z)))
                                    : dot_fma(Rk[0], x3, Rk[1], z, Rk[2], -y3);
            o[k] = (float)y;
        }
        if (a.rgb) {
            const uint8_t *c = a.rgb + 3 * ((size_t)f * HW + (size_t)v * a.width + u);
#pragma unroll
            for (int k = 0; k < 3; ++k) o[3 + k] = __fdiv_rn((float)c[k], 255.f);
        } else {
#pragma unroll
            for (int k = 0; k < 3; ++k) o[3 + k] = 0.f;
        }
    }
}

// ------------------------------------------------------------------------------------------------ host side
static int sd_tiles(const fcn_sunrgbd_depth_args *a) {
    return (int)(((long long)a->height * a->width + SD_TILE - 1) / SD_TILE);
}

static cudaError_t sd_layout(const fcn_sunrgbd_depth_args *a, Carve &c, SdWs &s) {
    const size_t F = (size_t)a->num_frames;
    s.tiles = (int32_t *)c.take(F * sd_tiles(a) * 4);
    s.total = (int32_t *)c.take(F * 4);
    return cudaSuccess;
}

// the capacities, which alone size the workspace
static int sd_check_sizes(const fcn_sunrgbd_depth_args *a, const char *fn) {
    if (a == nullptr) return invalid(fn, "NULL args");
    const long long F = a->num_frames, H = a->height, W = a->width, P = a->point_capacity;
    if (F < 1 || H < 1 || W < 1 || P < 1) return invalid(fn, "capacities must be >= 1");
    if (F > 65535 || H * W > (1LL << 30)) return invalid(fn, "too large (F <= 65535, H * W <= 2^30)");
    return FCN_OK;
}

static int sd_check(const fcn_sunrgbd_depth_args *a, const char *fn) {
    const int st = sd_check_sizes(a, fn);
    if (st != FCN_OK) return st;
    if (!a->depth || !a->image_hw || !a->calibs || !a->status) return invalid(fn, "NULL input");
    if (!a->clouds || !a->counts) return invalid(fn, "NULL output");
    if (((uintptr_t)a->depth & 1) != 0 || ((uintptr_t)a->calibs & 7) != 0 || ((uintptr_t)a->clouds & 3) != 0)
        return invalid(fn, "depth, calibs and clouds must be 2-, 8- and 4-byte aligned");
    return FCN_OK;
}

}  // namespace fcn

using namespace fcn;

extern "C" long long fcn_sunrgbd_depth_cloud_workspace_bytes(const fcn_sunrgbd_depth_args *a) {
    if (sd_check_sizes(a, __func__) != FCN_OK) return -1;
    SdWs s;
    return workspace_size(__func__, [&](Carve &c) { return sd_layout(a, c, s); });
}

extern "C" int fcn_sunrgbd_depth_cloud(const fcn_sunrgbd_depth_args *a, fcn_stream_t stream) {
    int st = sd_check(a, __func__);
    if (st != FCN_OK) return st;
    SdWs s;
    st = carve_workspace(__func__, "sunrgbd_depth_cloud", a->workspace, a->workspace_bytes,
                         [&](Carve &c) { return sd_layout(a, c, s); });
    if (st != FCN_OK) return st;
    cudaStream_t cs = (cudaStream_t)stream;
    const int F = a->num_frames, C = sd_tiles(a);
    sd_count_kernel<<<dim3(C, F), SD_THREADS, 0, cs>>>(*a, s, C);
    FCN_LAUNCH_CHECK();
    sd_scan_kernel<<<F, SD_THREADS, 0, cs>>>(*a, s, C);
    FCN_LAUNCH_CHECK();
    sd_write_kernel<<<dim3(C, F), SD_THREADS, 0, cs>>>(*a, s, C);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}
