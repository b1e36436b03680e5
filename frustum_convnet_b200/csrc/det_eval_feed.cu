// The evaluators' inputs built from the detection collector's device rows (C ABI section (19)): the KITTI result
// records of write_detection_results (train/test_net_det.py:88-123) and the SUN-RGBD corners of compute_box_3d
// (datasets/data_utils.py:44-70), written straight into the per-image / per-class order fcn_kitti_eval_* and
// fcn_sunrgbd_eval_* read, with no host pass over the rows.
//
// One thread per row the collector counted (fcn_det_prepare's seg_offsets[S]): it finds its segment s by binary
// search over seg_offsets, skips the row unless it is one of the keep_count[s] kept rows and seg_dst[s] >= 0, and
// writes output record seg_dst[s] + k.  The host derives seg_dst from the segment keys alone (the gather order of the
// dict path), so the order of the outputs is decided on the host and every row lands in one fixed slot.
//
// Exactness.  The quantization of '%.4f' / '%f' is exact: a float32 times 10^4 or 10^6 is exact in float64, so
// rint (ties to even) and one IEEE division give the double strtod reads back (kitti_eval.quantize); the products and
// the division use __dmul_rn / __ddiv_rn so that contraction cannot touch them.  atan2, cos and sin are computed in
// float64 and rounded once to float32: the correctly rounded float32 value, where numpy's float32 SIMD loops differ
// from it in the last bit on a share of inputs that depends on the CPU.  The rest of alpha and of the corners follows
// numpy's evaluation order, every operation rounded on its own.
#include <cmath>

#include "common.cuh"
#include "det_quantize.cuh"

namespace fcn {

constexpr int DF_THREADS = 256;
constexpr float DF_PI_F = 3.14159265358979323846f;      // np.pi as numpy casts it into a float32 expression

// the segment of counted row r: the last s with seg_offsets[s] <= r (empty segments skipped)
__device__ __forceinline__ int df_segment_of(const int32_t *__restrict__ off, int num_segments, int r) {
    int lo = 0, hi = num_segments - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= r) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// the output record of counted row r, or -1 when the row is not kept or its segment is not written
__device__ __forceinline__ int df_destination(const fcn_det_eval_feed_args &a, int r, int &s) {
    s = df_segment_of(a.seg_offsets, a.num_segments, r);
    const int k = r - a.seg_offsets[s];
    const int dst = a.seg_dst[s];
    return (dst < 0 || k >= a.keep_count[s]) ? -1 : dst + k;
}

// compute_alpha (datasets/provider_sample.py:389-394) in numpy's float32 order: (-sign(b) * pi) / 2 + b + ry
__device__ __forceinline__ float df_alpha(float x, float z, float ry) {
    const float b = (float)atan2((double)z, (double)x);
    const float sg = b > 0.f ? 1.f : (b < 0.f ? -1.f : (b == 0.f ? 0.f : b));     // np.sign: +0 for either zero
    const float t = __fdiv_rn(__fmul_rn(-sg, DF_PI_F), 2.f);
    return __fadd_rn(__fadd_rn(t, b), ry);
}

__global__ void __launch_bounds__(DF_THREADS) df_kitti_kernel(fcn_det_eval_feed_args a) {
    const int r = blockIdx.x * DF_THREADS + threadIdx.x;
    if (r >= a.num_rows) return;
    int s;
    const int o = df_destination(a, r, s);
    if (o < 0) return;
    // row [x1, y1, x2, y2, tx, ty, tz, h, w, l, ry, score] -> [code, alpha, x1, y1, x2, y2, h, w, l, tx, ty, tz, ry,
    // score] (FCN_KITTI_DET_COLS)
    const float *__restrict__ row = a.rows + (size_t)r * 12;
    float v[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) v[i] = row[i];
    double *__restrict__ out = a.records + (size_t)o * FCN_KITTI_DET_COLS;
    out[0] = (double)a.seg_value[s];
    out[1] = df_quantize(df_alpha(v[4], v[6], v[10]), 1e4);
#pragma unroll
    for (int i = 0; i < 4; ++i) out[2 + i] = df_quantize(v[i], 1e4);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        out[6 + i] = df_quantize(v[7 + i], 1e4);
        out[9 + i] = df_quantize(v[4 + i], 1e4);
    }
    out[12] = df_quantize(v[10], 1e4);
    out[13] = df_quantize(v[11], 1e6);
}

__global__ void __launch_bounds__(DF_THREADS) df_sunrgbd_kernel(fcn_det_eval_feed_args a) {
    const int r = blockIdx.x * DF_THREADS + threadIdx.x;
    if (r >= a.num_rows) return;
    int s;
    const int o = df_destination(a, r, s);
    if (o < 0) return;
    // row [x1, y1, x2, y2, tx, ty, tz, l, w, h, ry, score]; compute_box_3d: float32 cos / sin and half sizes, then
    // the rotation about y and the translation in float64
    const float *__restrict__ row = a.rows + (size_t)r * 12;
    const float ry = row[10];
    const double c = (double)(float)cos((double)ry), sn = (double)(float)sin((double)ry);
    const double hl = (double)__fdiv_rn(row[7], 2.f), hw = (double)__fdiv_rn(row[8], 2.f);
    const double hh = (double)__fdiv_rn(row[9], 2.f);
    const double tx = row[4], ty = row[5], tz = row[6];
    double *__restrict__ out = a.corners + (size_t)o * 24;
    bool finite = true;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const double xc = (i & 2) ? -hl : hl;                       // sx = [1, 1, -1, -1, 1, 1, -1, -1]
        const double yc = i < 4 ? hh : -hh;                         // sy = [1, 1, 1, 1, -1, -1, -1, -1]
        const double zc = ((i + 1) & 2) ? -hw : hw;                 // sz = [1, -1, -1, 1, 1, -1, -1, 1]
        const double x = __dadd_rn(__dadd_rn(__dmul_rn(c, xc), __dmul_rn(sn, zc)), tx);
        const double y = __dadd_rn(yc, ty);
        const double z = __dadd_rn(__dadd_rn(__dmul_rn(-sn, xc), __dmul_rn(c, zc)), tz);
        out[3 * i + 0] = x;
        out[3 * i + 1] = y;
        out[3 * i + 2] = z;
        finite = finite && isfinite(x) && isfinite(y) && isfinite(z);
    }
    const double score = row[11];
    a.scores[o] = score;
    a.segments[o] = a.seg_value[s];
    if (a.status != nullptr && !(finite && isfinite(score))) atomicOr(a.status, FCN_DET_FEED_NONFINITE);
}

// Host-side checks shared by both entries: counts, pointers, the collector's offsets and the gather plan.
static int df_check(const fcn_det_eval_feed_args *a, const char *fn) {
    if (a == nullptr) return invalid(fn, "NULL args");
    const int S = a->num_segments;
    if (S < 0 || a->num_rows < 0 || a->num_out < 0)
        return invalid(fn, "negative count (num_segments, num_rows, num_out must be >= 0)");
    if (a->num_out > (1 << 28)) return invalid(fn, "too many output records (num_out <= 2^28)");
    if (!a->host_seg_offsets || !a->host_keep_count || !a->host_seg_dst) return invalid(fn, "NULL host copies");
    if (!offsets_ok(a->host_seg_offsets, S, a->num_rows))
        return invalid(fn, "seg_offsets must start at 0, never decrease and end at num_rows");
    long long written = 0;
    for (int s = 0; s < S; ++s) {
        const int kc = a->host_keep_count[s], dst = a->host_seg_dst[s];
        if (kc < 0 || kc > a->host_seg_offsets[s + 1] - a->host_seg_offsets[s])
            return invalid(fn, "keep_count[s] must lie in [0, seg_offsets[s+1] - seg_offsets[s]]");
        if (dst < -1 || (dst >= 0 && (long long)dst + kc > a->num_out))
            return invalid(fn, "seg_dst[s] must be -1 or leave its kept rows inside [0, num_out)");
        if (dst >= 0) written += kc;
    }
    if (written != a->num_out) return invalid(fn, "the kept rows of the written segments must add up to num_out");
    if (a->num_rows > 0 && S > 0 && (!a->rows || !a->seg_offsets || !a->keep_count || !a->seg_dst || !a->seg_value))
        return invalid(fn, "NULL pointer");
    return FCN_OK;
}

static int df_launch(const fcn_det_eval_feed_args *a, void (*kern)(fcn_det_eval_feed_args), fcn_stream_t stream) {
    if (a->num_rows == 0 || a->num_segments == 0 || a->num_out == 0) return FCN_OK;
    kern<<<ceil_div(a->num_rows, DF_THREADS), DF_THREADS, 0, (cudaStream_t)stream>>>(*a);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

}  // namespace fcn

using namespace fcn;

extern "C" int fcn_det_kitti_records(const fcn_det_eval_feed_args *a, fcn_stream_t stream) {
    const int st = df_check(a, __func__);
    if (st != FCN_OK) return st;
    if (a->num_out > 0 && !a->records) return invalid(__func__, "NULL records");
    return df_launch(a, df_kitti_kernel, stream);
}

extern "C" int fcn_det_sunrgbd_feed(const fcn_det_eval_feed_args *a, fcn_stream_t stream) {
    const int st = df_check(a, __func__);
    if (st != FCN_OK) return st;
    if (a->num_out > 0 && (!a->corners || !a->scores || !a->segments))
        return invalid(__func__, "NULL corners, scores or segments");
    return df_launch(a, df_sunrgbd_kernel, stream);
}
