// fcn_frame_store_append (C ABI section (25)): one frame call's kept rows appended to a device store, with every size
// read on the device, so the append is captured in the same CUDA graph as the stage it follows.  In order:
//   fs_plan   one CTA: the call's segments (seg_class >= 0, ids[f] >= 0) counted and their rows summed, the whole-call
//             capacity decision against the cursor, then (when the call fits) the segment table written at the
//             cursor with a block scan of the keep counts, each segment's source offset kept in the workspace, the
//             call's bases kept in the workspace plan and the cursor advanced;
//   fs_copy   a grid over the call's row capacity: each thread moves one 16-byte third of a row, finding its store
//             segment by binary search over the offsets just written; threads past the call's rows exit.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace fcn {

constexpr int FS_THREADS = 256;
constexpr int FS_COPY_THREADS = 256;
constexpr int FS_QUADS = 3;                         // float4 pieces of a 12-float row

struct FsPlan {
    int32_t seg_base, row_base, segments, rows;     // the call's place in the store and its size
    int32_t stored;                                 // 1 when the call was appended
};

struct FsWs {
    FsPlan *plan;
    int32_t *src;               // (S) source offset of the call's j-th appended segment
};

// segment s of the call: appended or not, its source offset and row count cut to [0, num_rows)
__device__ __forceinline__ bool fs_segment(const fcn_frame_store_args &a, int s, int &off, int &keep) {
    const int f = s / a.num_classes;
    off = 0;
    keep = 0;
    if (a.seg_class[s] < 0 || a.ids[f] < 0) return false;
    off = min(max(a.seg_offsets[s], 0), a.num_rows);
    keep = min(max(a.keep_count[s], 0), a.num_rows - off);
    return true;
}

__global__ void __launch_bounds__(FS_THREADS) fs_plan_kernel(const fcn_frame_store_args a, FsWs w) {
    using Scan = cub::BlockScan<int, FS_THREADS>;
    using Reduce = cub::BlockReduce<long long, FS_THREADS>;
    __shared__ union {
        typename Scan::TempStorage scan;
        typename Reduce::TempStorage reduce;
    } tmp;
    __shared__ int n_seg, n_row, seg_base, row_base, stored;
    const int S = a.num_frames * a.num_classes;
    // the call's size, in 64 bits: each row count is cut to num_rows, S of them may pass 2^31
    long long segs = 0, rows = 0;
    for (int s = threadIdx.x; s < S; s += FS_THREADS) {
        int off, keep;
        if (fs_segment(a, s, off, keep)) {
            ++segs;
            rows += keep;
        }
    }
    segs = Reduce(tmp.reduce).Sum(segs);
    __syncthreads();
    rows = Reduce(tmp.reduce).Sum(rows);
    if (threadIdx.x == 0) {
        fcn_frame_store_cursor *c = a.cursor;
        const bool seg_fit = c->segments >= 0 && segs <= (long long)a.segment_capacity - c->segments;
        const bool row_fit = c->rows >= 0 && rows <= (long long)a.row_capacity - c->rows;
        FsPlan p;
        p.seg_base = seg_base = c->segments;
        p.row_base = row_base = c->rows;
        p.stored = stored = seg_fit && row_fit;
        p.segments = n_seg = stored ? (int)segs : 0;
        p.rows = n_row = stored ? (int)rows : 0;
        *w.plan = p;
        if (!stored) c->status |= (seg_fit ? 0 : FCN_STORE_SEGMENTS) | (row_fit ? 0 : FCN_STORE_ROWS);
    }
    __syncthreads();
    if (!stored) return;
    const int calls = a.cursor->calls;
    int seg_run = 0, row_run = 0;
    for (int s0 = 0; s0 < S; s0 += FS_THREADS) {
        const int s = s0 + threadIdx.x;
        int off = 0, keep = 0;
        const bool app = s < S && fs_segment(a, s, off, keep);
        int j, r, nj, nr;
        Scan(tmp.scan).ExclusiveSum(app ? 1 : 0, j, nj);
        __syncthreads();
        Scan(tmp.scan).ExclusiveSum(keep, r, nr);
        __syncthreads();
        if (app) {
            const int f = s / a.num_classes;
            const int d = seg_base + seg_run + j;
            a.store_image[d] = a.ids[f];
            a.store_class[d] = a.seg_class[s];
            a.store_frame[d] = (int32_t)((unsigned)calls * (unsigned)a.num_frames + (unsigned)f);
            a.store_offset[d] = row_base + row_run + r;
            a.store_keep[d] = keep;
            w.src[seg_run + j] = off;
        }
        seg_run += nj;
        row_run += nr;
    }
    if (threadIdx.x == 0) {
        fcn_frame_store_cursor *c = a.cursor;
        a.store_offset[seg_base + n_seg] = row_base + n_row;
        c->segments = seg_base + n_seg;
        c->rows = row_base + n_row;
        c->calls = calls + 1;
        c->frame_status |= *a.status;
    }
}

// thread t: the 16-byte piece t % 3 of the call's row t / 3; grid over num_rows * 3
__global__ void __launch_bounds__(FS_COPY_THREADS) fs_copy_kernel(const fcn_frame_store_args a, FsWs w) {
    const FsPlan p = *w.plan;
    const long long t = (long long)blockIdx.x * FS_COPY_THREADS + threadIdx.x;
    const int i = (int)(t / FS_QUADS), q = (int)(t - (long long)i * FS_QUADS);
    if (i >= p.rows) return;
    const int dst = p.row_base + i;
    // the last of the call's segments whose first row is <= dst: zero-keep segments share their successor's offset
    int lo = 0, hi = p.segments - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (a.store_offset[p.seg_base + mid] <= dst) lo = mid;
        else hi = mid - 1;
    }
    const int src = w.src[lo] + (dst - a.store_offset[p.seg_base + lo]);
    const float4 *from = reinterpret_cast<const float4 *>(a.rows) + (size_t)src * FS_QUADS + q;
    float4 *to = reinterpret_cast<float4 *>(a.store_rows) + (size_t)dst * FS_QUADS + q;
    *to = *from;
}

// ------------------------------------------------------------------------------------------------ host side
static cudaError_t fs_layout(const fcn_frame_store_args *a, Carve &c, FsWs &w) {
    w.plan = (FsPlan *)c.take(sizeof(FsPlan));
    w.src = (int32_t *)c.take((size_t)a->num_frames * a->num_classes * 4);
    return cudaSuccess;
}

// the call's shape, which alone sizes the workspace
static int fs_check_sizes(const fcn_frame_store_args *a, const char *fn) {
    if (a == nullptr) return invalid(fn, "NULL args");
    if (a->num_frames < 1 || a->num_classes < 1 || a->num_rows < 1 || a->row_capacity < 1 || a->segment_capacity < 1)
        return invalid(fn, "num_frames, num_classes, num_rows and both capacities must be >= 1");
    if (a->num_frames > FCN_STORE_MAX_FRAMES || a->num_classes > FCN_STORE_MAX_CLASSES)
        return invalid(fn, "num_frames or num_classes out of range (<= FCN_STORE_MAX_FRAMES, FCN_STORE_MAX_CLASSES)");
    return FCN_OK;
}

static int fs_check(const fcn_frame_store_args *a, const char *fn) {
    const int st = fs_check_sizes(a, fn);
    if (st != FCN_OK) return st;
    if (!a->rows || !a->seg_offsets || !a->keep_count || !a->seg_class || !a->status || !a->ids)
        return invalid(fn, "NULL input");
    if (!a->store_rows || !a->store_image || !a->store_class || !a->store_frame || !a->store_offset ||
        !a->store_keep || !a->cursor)
        return invalid(fn, "NULL store");
    if (((uintptr_t)a->rows & 15) != 0 || ((uintptr_t)a->store_rows & 15) != 0)
        return invalid(fn, "rows and store_rows must be 16-byte aligned");
    return FCN_OK;
}

}  // namespace fcn

using namespace fcn;

extern "C" long long fcn_frame_store_append_workspace_bytes(const fcn_frame_store_args *a) {
    if (fs_check_sizes(a, __func__) != FCN_OK) return -1;
    FsWs w;
    return workspace_size(__func__, [&](Carve &c) { return fs_layout(a, c, w); });
}

extern "C" int fcn_frame_store_append(const fcn_frame_store_args *a, fcn_stream_t stream) {
    int st = fs_check(a, __func__);
    if (st != FCN_OK) return st;
    FsWs w;
    st = carve_workspace(__func__, "frame_store_append", a->workspace, a->workspace_bytes,
                         [&](Carve &c) { return fs_layout(a, c, w); });
    if (st != FCN_OK) return st;
    cudaStream_t cs = (cudaStream_t)stream;
    fs_plan_kernel<<<1, FS_THREADS, 0, cs>>>(*a, w);
    FCN_LAUNCH_CHECK();
    const int blocks = (int)(((long long)a->num_rows * FS_QUADS + FS_COPY_THREADS - 1) / FS_COPY_THREADS);
    fs_copy_kernel<<<blocks, FS_COPY_THREADS, 0, cs>>>(*a, w);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}
