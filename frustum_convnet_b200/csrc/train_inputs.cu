// Device-side training-batch builder (C ABI section 11): what ProviderDataset.__getitem__ of
// datasets/provider_sample.py (train branch), datasets/provider_sample_refine.py and
// datasets/provider_sample_sunrgbd.py (train and from_rgb_detection branches) compute per item on DataLoader workers,
// plus the collate (default_collate / refine collate_fn with edge padding), for a whole batch in one launch.  One CTA
// per batch item.
//
// Per-frustum values that never change (rotation cos/sin, GT box in the frame of the inputs, the refine predicted
// box's face means and arange start/step) come from the host, computed once with numpy's own expressions.  Everything
// that depends on the step's draws is done here in float64 with each product and sum rounded separately
// (__dmul_rn / __dadd_rn), as numpy rounds its elementwise expressions.  The rotations of rotate_pc_along_y go
// through BLAS in the reference (np.dot), which may fuse them; results then differ by at most one float32 ulp.
// The SUN-RGBD kind follows BLAS's order instead (see dot_fma): its frustum angle is the angle of the box-2D centre's
// own ray, so the refs' centre-view x is a cancellation down to ~1e-17 m, whose rounding noise a float32 ulp bar sees.
#include "common.cuh"
#include "input_builder.cuh"

namespace fcn {
namespace {

constexpr int kThreads = 256;
constexpr double kPi = 3.141592653589793;

__device__ __forceinline__ double dsub(double a, double b) { return __dadd_rn(a, -b); }
__device__ __forceinline__ double clip(double v, double lo, double hi) { return fmin(fmax(v, lo), hi); }

// rotate_pc_along_y's np.dot(pc[:, [0, 2]], rotmat.T) in that order: x' = x c + z (-s), z' = x s + z c
__device__ __forceinline__ void rotate_y_fma(double x, double z, double cs, double sn, double *xo, double *zo) {
    *xo = dot_fma(x, cs, z, -sn);
    *zo = dot_fma(x, sn, z, cs);
}

struct Item {
    const fcn_train_frustum *fr;
    bool flip;
    double shift, height, c[3], heading;   // GT centre / heading after flip and shifts
};

// ref centre t (< T[s]) of scale s, flipped like the reference's ref1..ref4 (float64)
__device__ __forceinline__ void ref_point(const fcn_train_input_args &a, const Item &it, int s, int t, double *x,
                                          double *y, double *z) {
    const fcn_train_frustum &f = *it.fr;
    const double st = a.stride[s];
    if (a.kind == FCN_TRAIN_DET) {
        const RectProjection proj(f.box2d, f.P);
        const double zz = section_depth<true>(t, st);                        // np.arange(0, max_depth, s) + s / 2.
        double xx;
        proj.at(zz, &xx, y);                                                  // project_image_to_rect
        rotate_y<true>(xx, zz, f.cs, f.sn, x, z);                             // get_center_view
    } else if (a.kind == FCN_TRAIN_SUNRGBD) {
        // project_image_to_upright_camera: camera (x, y, z) -> depth (x, z, -y) -> Rtilt @ . -> (X, -Z, Y)
        const double *K = f.K, *R = f.Rtilt;
        const double zz = section_depth<true>(t, st);
        const double xc = __dmul_rn(dsub(f.cx, K[2]), zz) / K[0];
        const double yc = -(__dmul_rn(dsub(f.cy, K[5]), zz) / K[4]);
        auto row = [&](int i) { return dot_fma(R[3 * i], xc, R[3 * i + 1], zz, R[3 * i + 2], yc); };
        *y = -row(2);
        rotate_y_fma(row(0), row(1), f.cs, f.sn, x, z);                       // get_center_view
    } else {
        // cz = np.arange(z1, z2, s) + s / 2.;  c{x,y} = (cz - c1[2]) / delta[2] * delta[{0,1}] + c1[{0,1}]
        *z = __dadd_rn(__dadd_rn(f.z_start, __dmul_rn((double)t, f.z_step[s])), st / 2.);
        const double q = dsub(*z, f.line0[2]) / f.line_delta[2];
        *x = __dadd_rn(__dmul_rn(q, f.line_delta[0]), f.line0[0]);
        *y = __dadd_rn(__dmul_rn(q, f.line_delta[1]), f.line0[1]);
    }
    if (it.flip) *x = -*x;
}

// generate_labels of one ref: 1 inside the half box, -1 inside the full box, 0 outside; *d = its distance to the centre
__device__ __forceinline__ int ref_label(const fcn_train_input_args &a, const Item &it, double hs, double hc, int t,
                                         double *d) {
    double x, y, z;
    ref_point(a, it, 1, t, &x, &y, &z);
    const double dx = dsub(x, it.c[0]), dy = dsub(y, it.c[1]), dz = dsub(z, it.c[2]);
    *d = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
    // compute_box_3d places corner k at roty(heading) @ (x_k, y_k, z_k) + centre: the box frame is R^T (p - c)
    const double lx = __dadd_rn(__dmul_rn(hc, dx), -__dmul_rn(hs, dz));
    const double lz = __dadd_rn(__dmul_rn(hs, dx), __dmul_rn(hc, dz));
    const double *sz = it.fr->size;
    const bool det = a.kind != FCN_TRAIN_REFINE;
    const double f1 = det ? 0.5 : 0.3, f2 = det ? 1.0 : 0.6;                  // dimension * 0.5 | 1  /  * 0.3 | 0.6
    auto inside = [&](double fac) {
        const double l = __dmul_rn(sz[0], fac) / 2., w = __dmul_rn(sz[1], fac) / 2., h = __dmul_rn(sz[2], fac) / 2.;
        return fabs(lx) <= l && fabs(dy) <= h && fabs(lz) <= w;
    };
    return inside(f1) ? 1 : (inside(f2) ? -1 : 0);
}

}  // namespace

// The collate widths of fcn_build_train_inputs_fixed, one per scale.
struct Widths {
    int32_t w[FCN_MAX_SCALES];
};

// B CTAs per launch (B = 32 in the reference cfgs) never fill the GPU, so occupancy is worth nothing here.  With
// minBlocks = 1 ptxas keeps the whole kernel in registers (74, no spills on sm_90a); without it, it picked 64
// registers and spilled once the SUN-RGBD projection was inlined.
// kFixed: each scale's collate width is widths.w[s] (fcn_build_train_inputs_fixed), not the batch's largest T.
template <bool kFixed>
__global__ void __launch_bounds__(kThreads, 1) build_train_inputs_kernel(const __grid_constant__ fcn_train_input_args a,
                                                                         const Widths widths) {
    const int b = blockIdx.x, tid = threadIdx.x;
    __shared__ int s_pad[FCN_MAX_SCALES];
    __shared__ double s_wd[kThreads / 32];
    __shared__ int s_wt[kThreads / 32];

    int fi = a.index[b];
    fi = fi < 0 ? 0 : (fi >= a.num_frustums ? a.num_frustums - 1 : fi);  // defensive clamp (validated on the host)
    Item it;
    it.fr = a.frustums + fi;
    const fcn_train_frustum &f = *it.fr;
    // ---- augmentation draws (:224-244 / :267-286) and the GT box they move
    it.flip = a.labels && a.random_flip && a.flip_u[b] > 0.5;
    it.c[0] = f.center[0], it.c[1] = f.center[1], it.c[2] = f.center[2], it.heading = f.heading;
    if (it.flip) it.c[0] = -it.c[0], it.heading = dsub(kPi, it.heading);
    it.shift = it.height = 0.0;
    const bool shifting = a.labels && a.random_shift;
    const bool sun = a.kind == FCN_TRAIN_SUNRGBD;
    if (shifting) {
        const double n = a.shift_n[b], dist = f.dist;
        if (a.kind != FCN_TRAIN_REFINE) {
            const double sh = clip(__dmul_rn(__dmul_rn(n, dist), 0.2), -0.5 * dist, 0.5 * dist);
            it.shift = dsub(clip(__dadd_rn(sh, it.c[2]), 0.0, a.max_depth), it.c[2]);
        } else {
            const double s1 = a.stride[0];
            it.shift = clip(__dmul_rn(__dmul_rn(n, dist), 0.1), -s1 * 2, 2 * s1);
        }
        it.c[2] = __dadd_rn(it.c[2], it.shift);
        if (sun) {                                                            // np.random.random() * 0.4 - 0.2
            it.height = dsub(__dmul_rn(a.height_u[b], 0.4), 0.2);
            it.c[1] = __dadd_rn(it.c[1], it.height);
        }
    }
    // ---- collate width of every scale: the batch's largest T (edge padding beyond an item's own T)
    if (tid < a.num_scales) {
        if constexpr (kFixed) {
            s_pad[tid] = widths.w[tid];
        } else {
            int m = 1;
            for (int i = 0; i < a.B; ++i) {
                int g = a.index[i];
                g = g < 0 ? 0 : (g >= a.num_frustums ? a.num_frustums - 1 : g);
                m = max(m, a.frustums[g].T[tid]);
            }
            s_pad[tid] = m;
        }
    }

    // ---- resampled point cloud (B,3,N) and seg labels (B,N)
    const long long p0 = a.point_offsets[fi];
    const int n_raw = (int)(a.point_offsets[fi + 1] - p0);
    float *pc = a.point_cloud + (size_t)b * 3 * a.N;
    const bool refine = a.kind == FCN_TRAIN_REFINE;
    for (int j = tid; j < a.N; j += kThreads) {
        int i = a.choice[(size_t)b * a.N + j];
        i = i < 0 ? 0 : (i >= n_raw ? n_raw - 1 : i);
        double x = 0., y = 0., z = 0.;
        if (n_raw > 0) {
            const size_t k = 3 * (size_t)(p0 + i);
            if (a.points_f64) {
                const double *p = (const double *)a.points;
                x = p[k], y = p[k + 1], z = p[k + 2];
            } else {
                const float *p = (const float *)a.points;
                x = p[k], y = p[k + 1], z = p[k + 2];
            }
        }
        if (refine) x = dsub(x, f.ref_center[0]), y = dsub(y, f.ref_center[1]), z = dsub(z, f.ref_center[2]);
        if (sun) rotate_y_fma(x, z, f.cs, f.sn, &x, &z);
        else rotate_y<true>(x, z, f.cs, f.sn, &x, &z);
        if (!a.points_f64) x = (float)x, y = (float)y, z = (float)z;       // written back into the dataset's dtype
        if (it.flip) x = -x;
        if (shifting) z = __dadd_rn(z, it.shift);
        // a Python float added to a float32 array is added in float32
        if (shifting && sun) y = a.points_f64 ? __dadd_rn(y, it.height) : (double)__fadd_rn((float)y, (float)it.height);
        pc[j] = (float)x;
        pc[a.N + j] = (float)y;
        pc[2 * a.N + j] = (float)z;
        if (a.seg_label != nullptr) a.seg_label[(size_t)b * a.N + j] = n_raw > 0 ? (long long)a.seg[p0 + i] : 0;
    }
    __syncthreads();

    // ---- section centres of every scale, edge padded to the batch width
    for (int s = 0; s < a.num_scales; ++s) {
        const int T = f.T[s], P = s_pad[s];
        float *c = a.centers[s] + (size_t)b * 3 * P;
        for (int t = tid; t < P; t += kThreads) {
            double x, y, z;
            ref_point(a, it, s, min(t, T - 1), &x, &y, &z);
            c[t] = (float)x;
            c[P + t] = (float)y;
            c[2 * P + t] = (float)z;
        }
    }

    if (a.labels) {
        // ---- cls_label on ref2: block-wide "any inside the half box" and first argmin of the distance
        double hs, hc;
        sincos(it.heading, &hs, &hc);
        const int T2 = f.T[1], P2 = s_pad[1];
        int any1 = 0;
        double bd = __longlong_as_double(0x7ff0000000000000LL);
        int bt = 0x7fffffff;
        for (int t = tid; t < T2; t += kThreads) {
            double d;
            any1 |= ref_label(a, it, hs, hc, t, &d) == 1;
            if (d < bd) bd = d, bt = t;                                        // t ascending: keeps the first minimum
        }
        for (int o = 16; o > 0; o >>= 1) {
            const double od = __shfl_down_sync(0xffffffffu, bd, o);
            const int ot = __shfl_down_sync(0xffffffffu, bt, o);
            if (od < bd || (od == bd && ot < bt)) bd = od, bt = ot;
        }
        if ((tid & 31) == 0) s_wd[tid >> 5] = bd, s_wt[tid >> 5] = bt;
        any1 = __syncthreads_or(any1);
        if (!any1) {
            bd = s_wd[0], bt = s_wt[0];
            for (int w = 1; w < kThreads / 32; ++w)
                if (s_wd[w] < bd || (s_wd[w] == bd && s_wt[w] < bt)) bd = s_wd[w], bt = s_wt[w];
        }
        long long *lab = a.cls_label + (size_t)b * P2;
        for (int t = tid; t < P2; t += kThreads) {
            const int te = min(t, T2 - 1);
            double d;
            int v = ref_label(a, it, hs, hc, te, &d);
            if (!any1 && te == bt) v = 1;
            lab[t] = v;
        }
    }

    // ---- per-item scalars
    if (tid == 0) {
        if (a.rot_angle != nullptr) a.rot_angle[b] = (float)f.rot;
        if (a.ref_center != nullptr)
            for (int k = 0; k < 3; ++k) a.ref_center[3 * b + k] = (float)f.ref_center[k];
        if (a.rgb_prob != nullptr) a.rgb_prob[b] = (float)f.rgb_prob;
        if (a.labels) {
            for (int k = 0; k < 3; ++k) {
                a.box3d_center[3 * b + k] = (float)it.c[k];
                a.box3d_size[3 * b + k] = (float)f.size[k];
            }
            a.box3d_heading[b] = (float)it.heading;
            a.size_class[b] = f.cls_index;
        }
    }
    if (a.one_hot != nullptr)
        for (int v = tid; v < a.num_classes; v += kThreads)
            a.one_hot[(size_t)b * a.num_classes + v] = f.cls_index == v ? 1.f : 0.f;
}

}  // namespace fcn

using namespace fcn;

// The checks both entries share; fn names the entry in the error.
#define TI_REQUIRE(cond, msg)                                   \
    do {                                                        \
        if (!(cond)) return invalid(fn, msg);                   \
    } while (0)
static int check_train_inputs(const fcn_train_input_args *args, const char *fn) {
    if (args == nullptr) return invalid(fn, "args is NULL");
    const fcn_train_input_args &a = *args;
    TI_REQUIRE(a.kind == FCN_TRAIN_DET || a.kind == FCN_TRAIN_REFINE || a.kind == FCN_TRAIN_SUNRGBD,
               "kind must be FCN_TRAIN_DET, FCN_TRAIN_REFINE or FCN_TRAIN_SUNRGBD");
    TI_REQUIRE(a.labels == 0 || a.labels == 1, "labels must be 0 or 1");
    TI_REQUIRE(a.kind != FCN_TRAIN_DET || a.labels == 1,
               "the detection provider's from_rgb_detection branch is fcn_build_inputs");
    TI_REQUIRE(a.rtc == 1, "only cfg.DATA.RTC = True is supported");
    TI_REQUIRE(a.extra_feat == 0, "only cfg.DATA.WITH_EXTRA_FEAT = False is supported");
    TI_REQUIRE(a.B >= 0 && a.N >= 1 && a.num_frustums >= 1, "bad sizes");
    TI_REQUIRE(a.num_scales >= 2 && a.num_scales <= FCN_MAX_SCALES, "num_scales must be in [2, FCN_MAX_SCALES]");
    TI_REQUIRE(a.num_classes >= 0 && a.num_classes <= 1024, "bad num_classes");
    for (int s = 0; s < a.num_scales; ++s) TI_REQUIRE(a.stride[s] > 0 && a.centers[s] != nullptr, "bad scale");
    TI_REQUIRE(a.kind != FCN_TRAIN_SUNRGBD || a.num_scales == 5, "the SUN-RGBD provider takes exactly 5 scales");
    TI_REQUIRE(a.kind == FCN_TRAIN_REFINE || a.max_depth > 0, "max_depth must be > 0");
    if (a.B == 0) return FCN_OK;
    TI_REQUIRE(a.points && a.point_offsets && a.frustums && a.index && a.choice && a.point_cloud && a.rot_angle,
               "NULL pointer");
    if (a.labels) {
        TI_REQUIRE(a.cls_label && a.box3d_center && a.box3d_heading && a.box3d_size && a.size_class,
                   "NULL label pointer");
        TI_REQUIRE((!a.random_flip || a.flip_u) && (!a.random_shift || a.shift_n), "NULL draw pointer");
    }
    TI_REQUIRE(a.kind == FCN_TRAIN_REFINE || !a.labels || (a.seg && a.seg_label), "detection needs seg and seg_label");
    TI_REQUIRE(a.kind != FCN_TRAIN_REFINE || a.ref_center, "refinement needs ref_center");
    TI_REQUIRE(a.kind == FCN_TRAIN_DET || a.labels || a.rgb_prob, "from_rgb_detection needs rgb_prob");
    TI_REQUIRE(a.kind != FCN_TRAIN_SUNRGBD || !a.labels || !a.random_shift || a.height_u,
               "the SUN-RGBD shift needs height_u");
    return FCN_OK;
}
#undef TI_REQUIRE

extern "C" int fcn_build_train_inputs(const fcn_train_input_args *args, fcn_stream_t stream) {
    const int st = check_train_inputs(args, __func__);
    if (st != FCN_OK || args->B == 0) return st;
    build_train_inputs_kernel<false><<<args->B, kThreads, 0, (cudaStream_t)stream>>>(*args, Widths{});
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}

extern "C" int fcn_build_train_inputs_fixed(const fcn_train_input_args *args, const int32_t *widths,
                                            fcn_stream_t stream) {
    const int st = check_train_inputs(args, __func__);
    if (st != FCN_OK) return st;
    if (widths == nullptr) return invalid(__func__, "NULL widths");
    Widths w{};
    for (int s = 0; s < args->num_scales; ++s) {
        if (widths[s] < 1) return invalid(__func__, "widths must be >= 1");
        w.w[s] = widths[s];
    }
    if (args->B == 0) return FCN_OK;
    build_train_inputs_kernel<true><<<args->B, kThreads, 0, (cudaStream_t)stream>>>(*args, w);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}
