// The float64 "point in 3-D box" test shared by the KITTI refinement extractor (csrc/refine_extract.cu, section (16))
// and the first-stage ground-truth extractor (csrc/gt_extract.cu, section (17)), so both label exactly the same points.
#pragma once

#include "common.cuh"

namespace fcn {

// The half-space test of oracle/refine_extract.py (in_box): the point in the box's own frame, in float64, every
// product and sum rounded separately.  Substitutes for scipy's Delaunay(corners).find_simplex >= 0.
__device__ __forceinline__ bool box3d_contains(const fcn_refine_box &b, float4 p) {
    const double dx = __dsub_rn((double)p.x, b.center[0]);
    const double dy = __dsub_rn((double)p.y, b.center[1]);
    const double dz = __dsub_rn((double)p.z, b.center[2]);
    const double lx = __dsub_rn(__dmul_rn(b.cs, dx), __dmul_rn(b.sn, dz));
    const double lz = __dadd_rn(__dmul_rn(b.sn, dx), __dmul_rn(b.cs, dz));
    return fabs(lx) <= b.half[0] && fabs(dy) <= b.half[1] && fabs(lz) <= b.half[2];
}

}  // namespace fcn
