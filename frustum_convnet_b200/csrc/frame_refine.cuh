// Launchers of the section (16) and (20) kernels that fcn_frame_refine_extract (csrc/frame_refine.cu, section (22))
// runs unchanged over its F * J job slots.  Each launches the kernel as its own entry does.
#pragma once

#include "common.cuh"

namespace fcn {

// rj_jobs_kernel over a.num_jobs jobs (csrc/refine_jobs.cu)
cudaError_t rj_jobs(const fcn_refine_jobs_args &a, cudaStream_t s);

// rj_table_kernel over a.num_kept kept frustums (csrc/refine_jobs.cu)
cudaError_t rj_table(const fcn_refine_frustum_table_args &a, cudaStream_t s);

// rx_count_kernel in FCN_REFINE_DET mode over num_jobs jobs (csrc/refine_extract.cu)
cudaError_t rx_count_det(int num_frames, int num_jobs, const int32_t *so, const fcn_refine_box *jobs,
                         const int32_t *job_frame, const int32_t *pos, const float4 *fov_pts, int32_t *job_points,
                         int32_t *job_gt, int32_t *keep, long long *cnt, int32_t *bad, cudaStream_t s);

// rx_write_kernel without labels over num_jobs jobs (csrc/refine_extract.cu)
cudaError_t rx_write_det(int num_jobs, int num_kept, long long num_out, const int32_t *so, const fcn_refine_box *jobs,
                         const int32_t *job_frame, const int32_t *job_points, const int32_t *job_gt,
                         const int32_t *keep_pos, const long long *cnt_pos, const int32_t *pos, const float4 *fov_pts,
                         float4 *points, int32_t *offsets, cudaStream_t s);

}  // namespace fcn
