// The in-image point stage shared by the KITTI frustum extractors (csrc/frustum_extract.cu, section (15),
// csrc/refine_extract.cu, section (16), and csrc/gt_extract.cu, section (17)): each scan point projected velo -> rect
// -> image once in float64 and tested against the image (get_lidar_in_image_fov, draw_util.py:15-18), then the
// in-image points of every frame compacted in scan order.  The kernels of all three files call these bodies, so they
// extract exactly the same points.
#pragma once

#include "common.cuh"
#include "input_builder.cuh"

namespace fcn {

constexpr int FX_THREADS = 256;
constexpr int FX_FRAME_DOUBLES = 33;     // P (12), V2C (12), R0 (9) of fcn_frustum_frame

// velo (x, y, z) -> float32 rect and float64 image coordinates; true when the point is in the image.  The order of the
// operations is restated by oracle/frustum_extract.py.
__device__ __forceinline__ bool fx_project(const double *__restrict__ m, int height, int width, float4 s, float4 *rect,
                                           double *u, double *v) {
    const double *P = m, *V = m + 12, *R = m + 24;
    const double x = s.x, y = s.y, z = s.z;
    double ref[3], r[3], img[3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
        ref[i] = dadd<true>(dadd<true>(dadd<true>(dmul<true>(V[4 * i], x), dmul<true>(V[4 * i + 1], y)),
                                       dmul<true>(V[4 * i + 2], z)), V[4 * i + 3]);
#pragma unroll
    for (int i = 0; i < 3; ++i)
        r[i] = dadd<true>(dadd<true>(dmul<true>(R[3 * i], ref[0]), dmul<true>(R[3 * i + 1], ref[1])),
                          dmul<true>(R[3 * i + 2], ref[2]));
#pragma unroll
    for (int i = 0; i < 3; ++i)
        img[i] = dadd<true>(dadd<true>(dadd<true>(dmul<true>(P[4 * i], r[0]), dmul<true>(P[4 * i + 1], r[1])),
                                       dmul<true>(P[4 * i + 2], r[2])), P[4 * i + 3]);
    *u = __ddiv_rn(img[0], img[2]);
    *v = __ddiv_rn(img[1], img[2]);
    *rect = make_float4((float)r[0], (float)r[1], (float)r[2], s.w);
    return *u >= 0.0 && *u < (double)width && *v >= 0.0 && *v < (double)height && s.x > 2.0f;
}

// one frame per blockIdx.y; the frame's matrices in shared memory
__device__ __forceinline__ void fx_load_frame(const fcn_frustum_frame *__restrict__ frames, int f, double *m) {
    if (threadIdx.x < FX_FRAME_DOUBLES) m[threadIdx.x] = frames[f].P[threadIdx.x];   // P, V2C, R0 are contiguous
    __syncthreads();
}

// Body of a flag kernel: grid (points of the largest frame / FX_THREADS, frames), flags[i] = point i is in the image.
__device__ __forceinline__ void fov_flag(const float4 *__restrict__ scans, const int32_t *__restrict__ so,
                                         const fcn_frustum_frame *__restrict__ frames, int32_t *__restrict__ flags) {
    __shared__ double m[FX_FRAME_DOUBLES];
    const int f = blockIdx.y;
    fx_load_frame(frames, f, m);
    const int i = so[f] + blockIdx.x * FX_THREADS + threadIdx.x;
    if (i >= so[f + 1]) return;
    float4 rect;
    double u, v;
    flags[i] = fx_project(m, frames[f].height, frames[f].width, scans[i], &rect, &u, &v) ? 1 : 0;
}

// Body of a compact kernel (same grid): every in-image point, recomputed, stored at its exclusive-sum position pos[i]
// as float32 rect x, y, z and intensity, with its float64 image coordinates when kUV.
template <bool kUV>
__device__ __forceinline__ void fov_compact(const float4 *__restrict__ scans, const int32_t *__restrict__ so,
                                            const fcn_frustum_frame *__restrict__ frames,
                                            const int32_t *__restrict__ pos, float4 *__restrict__ fov_pts,
                                            double *__restrict__ fov_u, double *__restrict__ fov_v) {
    __shared__ double m[FX_FRAME_DOUBLES];
    const int f = blockIdx.y;
    fx_load_frame(frames, f, m);
    const int i = so[f] + blockIdx.x * FX_THREADS + threadIdx.x;
    if (i >= so[f + 1]) return;
    float4 rect;
    double u, v;
    if (fx_project(m, frames[f].height, frames[f].width, scans[i], &rect, &u, &v)) {
        const int k = pos[i];
        fov_pts[k] = rect;
        if (kUV) {
            fov_u[k] = u;
            fov_v[k] = v;
        }
    }
}

// Host check of the scans both extractors take: 16-byte-aligned float4 points and the host copy of the scan offsets
// (num_frames + 1 entries).  Raises *max_n (0 on entry) to the largest scan, the x extent of the flag and compact
// grids.
inline int check_scans(const char *fn, const int32_t *host_so, int num_frames, int num_points, const void *scans,
                       int *max_n) {
    if (!host_so) return invalid(fn, "NULL host_scan_offsets");
    if (((uintptr_t)scans & 15) != 0) return invalid(fn, "scans must be 16-byte aligned");
    if (!offsets_ok(host_so, num_frames, num_points))
        return invalid(fn, "scan offsets must start at 0, never decrease and end at num_points");
    for (int f = 0; f < num_frames; ++f)
        if (host_so[f + 1] - host_so[f] > *max_n) *max_n = host_so[f + 1] - host_so[f];
    return FCN_OK;
}

}  // namespace fcn
