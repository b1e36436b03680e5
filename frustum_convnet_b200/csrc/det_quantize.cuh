// The text round trip of the collector's rows, shared by the evaluator feed (csrc/det_eval_feed.cu) and the refinement
// job table (csrc/refine_jobs.cu), so both read back exactly the values write_detection_results writes.
#pragma once

#include "common.cuh"

namespace fcn {

// '%.<d>f' then strtod of a float32 value, s = 10^d: a float32 times 10^4 or 10^6 is exact in float64, so rint (ties
// to even, as printf rounds an exact tie) and one IEEE division give the double strtod reads back
__device__ __forceinline__ double df_quantize(float v, double s) { return __ddiv_rn(rint(__dmul_rn((double)v, s)), s); }

}  // namespace fcn
