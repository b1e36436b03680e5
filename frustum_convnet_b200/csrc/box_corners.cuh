// Box corners and bounding-cube test of the rotated 3-D NMS (shared by nms3d.cu and detect.cu).
#pragma once

namespace fcn {

// corners in the reference order (rbbox_iou.py:131-147 == models/model_util.py:48-72)
__device__ __forceinline__ void box_to_corners(const float *d, float *c) {
    const float cx = d[0], cy = d[1], cz = d[2], l = d[3], w = d[4], h = d[5], r = d[6];
    const float cs = cosf(r), sn = sinf(r);
    const float xs[8] = {l / 2, l / 2, -l / 2, -l / 2, l / 2, l / 2, -l / 2, -l / 2};
    const float ys[8] = {h / 2, h / 2, h / 2, h / 2, -h / 2, -h / 2, -h / 2, -h / 2};
    const float zs[8] = {w / 2, -w / 2, -w / 2, w / 2, w / 2, -w / 2, -w / 2, w / 2};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        c[3 * i + 0] = cs * xs[i] + sn * zs[i] + cx;
        c[3 * i + 1] = ys[i] + cy;
        c[3 * i + 2] = -sn * xs[i] + cs * zs[i] + cz;
    }
}

// standup IoU > 0 <=> the axis-aligned bounding cubes [min xyz, max xyz] overlap with positive volume
// (rbbox_iou.py:62-96, nms_cpu.h:192)
__device__ __forceinline__ bool cubes_overlap(const float *a, const float *b) {
    return fminf(a[3], b[3]) - fmaxf(a[0], b[0]) > 0.f && fminf(a[4], b[4]) - fmaxf(a[1], b[1]) > 0.f &&
           fminf(a[5], b[5]) - fmaxf(a[2], b[2]) > 0.f;
}

}  // namespace fcn
