// The frame kernels of fcn_frame_extract (csrc/frame_extract.cu), launched by its entry in csrc/frustum_extract.cu.
#pragma once

#include "common.cuh"

namespace fcn {

// frame_setup_kernel, then frame_pack_kernel: scan offsets so (F + 1), det_frame (F * D) and packed (F * P) filled
cudaError_t frame_setup(const fcn_frame_extract_args &a, int32_t *so, int32_t *det_frame, float4 *packed,
                        cudaStream_t s);

// frame_slots_kernel after the count pass: c2, kpos, base (F * D each) for the write kernel
cudaError_t frame_slots(const fcn_frame_extract_args &a, const int32_t *det_points, int32_t *c2, int32_t *kpos,
                        long long *base, cudaStream_t s);

}  // namespace fcn
