// The stages shared by the KITTI frustum extractors (csrc/frustum_extract.cu, section (15), csrc/refine_extract.cu,
// section (16), and csrc/gt_extract.cu, section (17)).  Each extractor's count entry runs
//   fov_stage    flag the in-image points, scan the flags, compact the in-image points (csrc/frustum_fov.cu);
//   its own count kernel, one CTA per job over the job's frame's in-image points (job_count, job_words here);
//   job_totals   scan the kept flags and the point counts, then the info words;
// and its write entry one CTA per kept job (kept_slot, job_scatter here).  The extractors differ only in their job
// tests, drop rules and per-frustum extras, so they extract exactly the same in-image points.
#pragma once

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace fcn {

constexpr int FX_THREADS = 256;

// Workspace pieces of the job pass (kept flags, point counts, their scans and the bad-reference counter), which
// every extractor has, the SUN-RGBD one (csrc/sunrgbd_extract.cu, section (18)) included.
struct JobWs {
    int32_t *keep, *keep_pos, *bad;
    long long *cnt, *cnt_pos;
    void *temp;
    size_t temp_bytes;
};

// Plus the in-image stage's pieces of the KITTI extractors; each family carves its own pieces after these.
struct FovWs : JobWs {
    int32_t *flags, *pos;
    float4 *fov_pts;
    double *fov_u, *fov_v;      // float64 image coordinates of the in-image points (null unless uv)
};

// Takes the job pieces for num_jobs jobs from c, with room in temp for at least min_temp_bytes.
cudaError_t job_carve(Carve &c, int num_jobs, size_t min_temp_bytes, JobWs &w);

// Takes the shared pieces for num_points scan points and num_jobs jobs from c (fov_u, fov_v only when uv).
cudaError_t fov_carve(Carve &c, int num_points, int num_jobs, bool uv, FovWs &w);

// The start of every count entry on stream s: clears the tails of the keep and cnt scans and the bad counter.
cudaError_t job_reset(const JobWs &w, int num_jobs, cudaStream_t s);

// The in-image stage of a count entry on stream s: clears the flag scan's tail, job_reset, then flags every scan
// point, scans the flags into pos and compacts the in-image points of each frame, in scan order, to fov_pts (and
// fov_u, fov_v).  max_n is the largest scan (check_scans), the x extent of the flag and compact grids.
cudaError_t fov_stage(const FovWs &w, int num_points, int num_jobs, int num_frames, int max_n, const void *scans,
                      const int32_t *scan_offsets, const fcn_frustum_frame *frames, cudaStream_t s);

// After the count kernel: exclusive sums over keep and cnt, then info = (kept jobs, their points, bad, 0).
cudaError_t job_totals(const JobWs &w, int num_jobs, long long *info, cudaStream_t s);

// One job's count over its frame's in-image points [p0, p1): visit(i, c, l) adds in-image point i to the thread's
// count c and, with kLabels, to its labelled count l.  The block's c and l end up on thread 0.
template <bool kLabels, typename Visit>
__device__ __forceinline__ void job_count(int p0, int p1, int &c, int &l, Visit visit) {
    using Reduce = cub::BlockReduce<int, FX_THREADS>;
    __shared__ typename Reduce::TempStorage tmp;
    c = 0;
    l = 0;
    for (int i = p0 + threadIdx.x; i < p1; i += FX_THREADS) visit(i, c, l);
    c = Reduce(tmp).Sum(c);
    if (kLabels) {
        __syncthreads();
        l = Reduce(tmp).Sum(l);
    }
}

// A count kernel's words for job j (thread 0): its point count c, kept, or -1 and not kept when dropped.
__device__ __forceinline__ void job_words(int j, bool drop, int c, int32_t *__restrict__ job_points,
                                          int32_t *__restrict__ keep, long long *__restrict__ cnt) {
    job_points[j] = drop ? -1 : c;
    keep[j] = drop ? 0 : 1;
    cnt[j] = drop ? 0 : c;
}

// The write kernel's guard for job j: false when the job was dropped (c < 0) or the sizes the host read disagree
// with the count pass; else its slot *k and first output position *base, with offsets[*k + 1] written.
__device__ __forceinline__ bool kept_slot(int j, int c, int num_kept, long long num_out,
                                          const int32_t *__restrict__ keep_pos, const long long *__restrict__ cnt_pos,
                                          int32_t *__restrict__ offsets, int *k, long long *base) {
    if (c < 0) return false;
    const int kj = keep_pos[j];
    const long long bj = cnt_pos[j];
    if (kj >= num_kept || bj + c > num_out) return false;
    if (threadIdx.x == 0) offsets[kj + 1] = (int32_t)(bj + c);
    *k = kj;
    *base = bj;
    return true;
}

// A write kernel's stable scatter: the in-image points i of [p0, p1) with in(i), in scan order, handed to put(o, i)
// at the output positions o = base, base + 1, ...; stops once the job's c points are placed.
template <typename In, typename Put>
__device__ __forceinline__ void job_scatter(int p0, int p1, int c, long long base, In in, Put put) {
    using Scan = cub::BlockScan<int, FX_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    int run = 0;
    for (int i0 = p0; i0 < p1 && run < c; i0 += FX_THREADS) {
        const int i = i0 + threadIdx.x;
        const int flag = i < p1 && in(i);
        int off, total;
        Scan(tmp).ExclusiveSum(flag, off, total);
        if (flag) put(base + run + off, i);
        run += total;
        __syncthreads();
    }
}

// Host check of the scans every extractor takes: points aligned to `align` bytes (16 for the KITTI float4 points, 4
// for SUN-RGBD's 6-float rows) and the host copy of the scan offsets (num_frames + 1 entries).  Raises *max_n (0 on
// entry) to the largest scan, the x extent of the flag and compact grids.
inline int check_scans(const char *fn, const int32_t *host_so, int num_frames, int num_points, const void *scans,
                       int align, int *max_n) {
    if (!host_so) return invalid(fn, "NULL host_scan_offsets");
    if (((uintptr_t)scans & (align - 1)) != 0) {
        char msg[32];
        snprintf(msg, sizeof(msg), "scans must be %d-byte aligned", align);
        return invalid(fn, msg);
    }
    if (!offsets_ok(host_so, num_frames, num_points))
        return invalid(fn, "scan offsets must start at 0, never decrease and end at num_points");
    for (int f = 0; f < num_frames; ++f)
        if (host_so[f + 1] - host_so[f] > *max_n) *max_n = host_so[f + 1] - host_so[f];
    return FCN_OK;
}

}  // namespace fcn
