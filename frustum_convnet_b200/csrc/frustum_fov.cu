// The in-image point stage and the job totals shared by the KITTI frustum extractors (frustum_fov.cuh): each scan
// point projected velo -> rect -> image once in float64 and tested against the image (get_lidar_in_image_fov,
// draw_util.py:15-18), then the in-image points of every frame compacted in scan order; after an extractor's count
// kernel, the exclusive sums over its kept jobs and their point counts.
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "frustum_fov.cuh"
#include "input_builder.cuh"

namespace fcn {

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

// grid (points of the largest frame / FX_THREADS, frames): flags[i] = point i is in the image
__global__ void __launch_bounds__(FX_THREADS)
fov_flag_kernel(const float4 *__restrict__ scans, const int32_t *__restrict__ so,
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

// Same grid: every in-image point, recomputed, stored at its exclusive-sum position pos[i] as float32 rect x, y, z
// and intensity, with its float64 image coordinates when kUV.
template <bool kUV>
__global__ void __launch_bounds__(FX_THREADS)
fov_compact_kernel(const float4 *__restrict__ scans, const int32_t *__restrict__ so,
                   const fcn_frustum_frame *__restrict__ frames, const int32_t *__restrict__ pos,
                   float4 *__restrict__ fov_pts, double *__restrict__ fov_u, double *__restrict__ fov_v) {
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

__global__ void job_info_kernel(int num_jobs, const int32_t *__restrict__ keep_pos,
                                const long long *__restrict__ cnt_pos, const int32_t *__restrict__ bad,
                                long long *__restrict__ info) {
    info[0] = keep_pos[num_jobs];
    info[1] = cnt_pos[num_jobs];
    info[2] = *bad;
    info[3] = 0;
}

cudaError_t job_carve(Carve &c, int num_jobs, size_t min_temp_bytes, JobWs &w) {
    const size_t J = (size_t)num_jobs;
    size_t t1 = 0, t2 = 0;
    cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, t1, (const int32_t *)nullptr, (int32_t *)nullptr,
                                                  num_jobs + 1);
    if (e != cudaSuccess) return e;
    e = cub::DeviceScan::ExclusiveSum(nullptr, t2, (const long long *)nullptr, (long long *)nullptr, num_jobs + 1);
    if (e != cudaSuccess) return e;
    w.temp_bytes = min_temp_bytes > t1 ? min_temp_bytes : t1;
    w.temp_bytes = w.temp_bytes > t2 ? w.temp_bytes : t2;
    w.keep = (int32_t *)c.take((J + 1) * 4);
    w.keep_pos = (int32_t *)c.take((J + 1) * 4);
    w.cnt = (long long *)c.take((J + 1) * 8);
    w.cnt_pos = (long long *)c.take((J + 1) * 8);
    w.bad = (int32_t *)c.take(4);
    w.temp = c.take(w.temp_bytes);
    return cudaSuccess;
}

cudaError_t fov_carve(Carve &c, int num_points, int num_jobs, bool uv, FovWs &w) {
    const size_t N = (size_t)num_points;
    size_t t0 = 0;
    cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, t0, (const int32_t *)nullptr, (int32_t *)nullptr,
                                                  num_points + 1);
    if (e != cudaSuccess) return e;
    w.flags = (int32_t *)c.take((N + 1) * 4);
    w.pos = (int32_t *)c.take((N + 1) * 4);
    w.fov_pts = (float4 *)c.take(N * 16);
    w.fov_u = uv ? (double *)c.take(N * 8) : nullptr;
    w.fov_v = uv ? (double *)c.take(N * 8) : nullptr;
    return job_carve(c, num_jobs, t0, w);
}

cudaError_t job_reset(const JobWs &w, int num_jobs, cudaStream_t s) {
    cudaError_t e;
    if ((e = cudaMemsetAsync(w.keep + num_jobs, 0, 4, s)) != cudaSuccess ||
        (e = cudaMemsetAsync(w.cnt + num_jobs, 0, 8, s)) != cudaSuccess)
        return e;
    return cudaMemsetAsync(w.bad, 0, 4, s);
}

cudaError_t fov_stage(const FovWs &w, int num_points, int num_jobs, int num_frames, int max_n, const void *scans,
                      const int32_t *scan_offsets, const fcn_frustum_frame *frames, cudaStream_t s) {
    cudaError_t e;
    if ((e = cudaMemsetAsync(w.flags + num_points, 0, 4, s)) != cudaSuccess ||
        (e = job_reset(w, num_jobs, s)) != cudaSuccess)
        return e;
    const float4 *pts = (const float4 *)scans;
    const dim3 grid(ceil_div(max_n, FX_THREADS), num_frames);
    if (max_n > 0) {
        fov_flag_kernel<<<grid, FX_THREADS, 0, s>>>(pts, scan_offsets, frames, w.flags);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    size_t temp_bytes = w.temp_bytes;
    e = cub::DeviceScan::ExclusiveSum(w.temp, temp_bytes, w.flags, w.pos, num_points + 1, s);
    if (e != cudaSuccess || max_n == 0) return e;
    if (w.fov_u)
        fov_compact_kernel<true><<<grid, FX_THREADS, 0, s>>>(pts, scan_offsets, frames, w.pos, w.fov_pts, w.fov_u,
                                                             w.fov_v);
    else
        fov_compact_kernel<false><<<grid, FX_THREADS, 0, s>>>(pts, scan_offsets, frames, w.pos, w.fov_pts, nullptr,
                                                              nullptr);
    return cudaGetLastError();
}

cudaError_t job_totals(const JobWs &w, int num_jobs, long long *info, cudaStream_t s) {
    size_t temp_bytes = w.temp_bytes;
    cudaError_t e = cub::DeviceScan::ExclusiveSum(w.temp, temp_bytes, w.keep, w.keep_pos, num_jobs + 1, s);
    if (e != cudaSuccess) return e;
    e = cub::DeviceScan::ExclusiveSum(w.temp, temp_bytes, w.cnt, w.cnt_pos, num_jobs + 1, s);
    if (e != cudaSuccess) return e;
    job_info_kernel<<<1, 1, 0, s>>>(num_jobs, w.keep_pos, w.cnt_pos, w.bad, info);
    return cudaGetLastError();
}

}  // namespace fcn
