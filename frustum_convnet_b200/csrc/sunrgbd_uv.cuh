// The SUN-RGBD image-plane arithmetic shared by the offline extractor (csrc/sunrgbd_extract.cu, section (18)) and the
// frame extractor (csrc/sunrgbd_frame.cu, section (23)), so both cut exactly the same in-box points.
#pragma once

#include "common.cuh"
#include "input_builder.cuh"

namespace fcn {

// project_upright_depth_to_image (sunrgbd_utils.py:109-123) of the point p = (x, y, z): d = Rtilt^T p, camera
// (d0, -d2, d1), (u, v, w) = K cam, every np.dot in dgemm's order (dot_fma), then u / w and v / w.  The same
// operations as sx_project_kernel, which keeps them written out: its SASS is pinned, and the inlined form changes
// its register allocation.
__device__ __forceinline__ void sx_project_point(const double *R, const double *K, double x, double y, double z,
                                                 double &u, double &v) {
    const double d0 = dot_fma(R[0], x, R[3], y, R[6], z);
    const double d1 = dot_fma(R[1], x, R[4], y, R[7], z);
    const double d2 = dot_fma(R[2], x, R[5], y, R[8], z);
    const double c0 = d0, c1 = -d2, c2 = d1;
    const double w = dot_fma(c0, K[6], c1, K[7], c2, K[8]);
    u = dot_fma(c0, K[0], c1, K[1], c2, K[2]) / w;
    v = dot_fma(c0, K[3], c1, K[4], c2, K[5]) / w;
}

// prepare_data.py:191-192, in its order: u < xmax, u >= xmin, v < ymax, v >= ymin (box: xmin, ymin, xmax, ymax)
__device__ __forceinline__ bool sx_in_uv_box(double u, double v, const double *box) {
    return u < box[2] && u >= box[0] && v < box[3] && v >= box[1];
}

}  // namespace fcn
