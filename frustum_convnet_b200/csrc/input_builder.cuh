// Per-frustum input math shared by the eval input builder (input_builder.cu) and the training-batch builder
// (train_inputs.cu): centre-view rotation (datasets/data_utils.py:7-21) and the section centres of generate_ref
// (datasets/provider_sample.py:291-327, data_utils.py:73-93).
// kExact = true rounds every product and sum separately (__dmul_rn / __dadd_rn), as numpy's elementwise float64
// expressions do; kExact = false is the plain expression the eval builder has always compiled (the compiler may
// contract it into FMAs), kept so that kernel's arithmetic does not change.
#pragma once

namespace fcn {

template <bool kExact>
__device__ __forceinline__ double dmul(double a, double b) {
    if constexpr (kExact) return __dmul_rn(a, b);
    else return a * b;
}
template <bool kExact>
__device__ __forceinline__ double dadd(double a, double b) {
    if constexpr (kExact) return __dadd_rn(a, b);
    else return a + b;
}

// x . y over k = 0, 1, 2 as OpenBLAS's dgemm accumulates it (numpy's np.dot of float64 matrices): a0 b0 rounded,
// then one FMA per further term.  Used by the SUN-RGBD training inputs (train_inputs.cu) and the SUN-RGBD frustum
// projection (sunrgbd_extract.cu).
__device__ __forceinline__ double dot_fma(double a0, double b0, double a1, double b1) {
    return __fma_rn(a1, b1, __dmul_rn(a0, b0));
}
__device__ __forceinline__ double dot_fma(double a0, double b0, double a1, double b1, double a2, double b2) {
    return __fma_rn(a2, b2, dot_fma(a0, b0, a1, b1));
}

// rot_angle = np.pi / 2.0 + frustum_angle  (provider_sample.py:330-333) and its sine / cosine
__device__ __forceinline__ double centre_view_angle(double frustum_angle, double *sn, double *cs) {
    const double rot = 1.5707963267948966 + frustum_angle;
    sincos(rot, sn, cs);
    return rot;
}

// pc[:, [0, 2]] = dot(pc[:, [0, 2]], rotmat.T), rotmat = [[c, -s], [s, c]]  ->  x' = x c - z s, z' = x s + z c
template <bool kExact>
__device__ __forceinline__ void rotate_y(double x, double z, double cs, double sn, double *xo, double *zo) {
    if constexpr (kExact) {
        *xo = __dadd_rn(__dmul_rn(x, cs), -__dmul_rn(z, sn));
        *zo = __dadd_rn(__dmul_rn(x, sn), __dmul_rn(z, cs));
    } else {
        *xo = x * cs - z * sn;
        *zo = x * sn + z * cs;
    }
}

// project_image_to_rect of the box-2D centre (cx, cy) at depth z with calib P (3x4 row-major)
struct RectProjection {
    double cx, cy, c_u, c_v, f_u, f_v, b_x, b_y;
    __device__ __forceinline__ RectProjection(const double *bx, const double *P) {
        cx = (bx[0] + bx[2]) / 2.0, cy = (bx[1] + bx[3]) / 2.0;
        c_u = P[2], c_v = P[6], f_u = P[0], f_v = P[5];
        b_x = P[3] / (-f_u), b_y = P[7] / (-f_v);
    }
    __device__ __forceinline__ void at(double z, double *x, double *y) const {
        *x = ((cx - c_u) * z) / f_u + b_x;
        *y = ((cy - c_v) * z) / f_v + b_y;
    }
};

// np.arange(0, max_depth, s)[t] + s / 2.
template <bool kExact>
__device__ __forceinline__ double section_depth(int t, double st) {
    return dadd<kExact>(dmul<kExact>((double)t, st), st / 2.0);
}

}  // namespace fcn
