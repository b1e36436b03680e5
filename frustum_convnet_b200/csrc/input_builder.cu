// Device-side input builder (SURVEY.md 8(f)-3): what datasets/provider_sample.py ProviderDataset.__getitem__ does
// per frustum on the host with numpy (4 DataLoader workers feeding ~12 KB/frustum), for a whole batch in one launch:
//   rot_angle = pi/2 + frustum_angle                                        (:330-333)
//   point_cloud[b,:,j] = rotate_pc_along_y(points_b[choice[b,j]], rot_angle) (:157-171,354-365; data_utils.py:7-21)
//   center_ref_s[b,:,t] = rotate(project_image_to_rect((cx, cy, t*stride + stride/2), P2), rot_angle)
//                                                                           (:173-182,291-327; data_utils.py:73-93)
//   one_hot[b, cls[b]] = 1                                                  (:148-151)
// The raw frustum points stay resident in HBM; per step only the resampling indices (the caller's RNG stream:
// np.random.choice with the reference's replace rule, :164-166) and a few scalars cross PCIe.
// Arithmetic is float64 with the float32 casts exactly where numpy makes them, so results are bit-identical to
// the reference up to the last-ulp difference between CUDA's and glibc's double sin/cos.
#include "common.cuh"
#include "input_builder.cuh"

namespace fcn {

__global__ void __launch_bounds__(256)
build_inputs_kernel(const __grid_constant__ fcn_input_args a) {
    const int b = blockIdx.x, tid = threadIdx.x;
    double sn, cs;
    const double rot = centre_view_angle(a.frustum_angle[b], &sn, &cs);
    if (tid == 0 && a.rot_angle != nullptr) a.rot_angle[b] = (float)rot;
    // ---- resampled, centre-view rotated point cloud (B,3,N)
    const float *pts = a.points + 3 * (size_t)a.point_offsets[b];
    const int n_raw = a.point_offsets[b + 1] - a.point_offsets[b];
    float *pc = a.point_cloud + (size_t)b * 3 * a.N;
    for (int j = tid; j < a.N; j += blockDim.x) {
        int i = a.choice[(size_t)b * a.N + j];
        i = i < 0 ? 0 : (i >= n_raw ? n_raw - 1 : i);               // defensive clamp (valid inputs are in range)
        double x, z;
        rotate_y<false>((double)pts[3 * i], (double)pts[3 * i + 2], cs, sn, &x, &z);
        pc[j] = (float)x;
        pc[a.N + j] = pts[3 * i + 1];
        pc[2 * a.N + j] = (float)z;
    }
    // ---- section centres of every scale
    const RectProjection proj(a.box2d + 4 * (size_t)b, a.P + 12 * (size_t)b);
    for (int s = 0; s < a.num_scales; ++s) {
        const int T = a.T[s];
        const double st = a.stride[s];
        float *c = a.centers[s] + (size_t)b * 3 * T;
        for (int t = tid; t < T; t += blockDim.x) {
            const double z = section_depth<false>(t, st);
            double x, y, xr, zr;
            proj.at(z, &x, &y);
            rotate_y<false>(x, z, cs, sn, &xr, &zr);
            c[t] = (float)xr;
            c[T + t] = (float)y;
            c[2 * T + t] = (float)zr;
        }
    }
    if (a.one_hot != nullptr)
        for (int v = tid; v < a.num_classes; v += blockDim.x)
            a.one_hot[(size_t)b * a.num_classes + v] = (a.cls_index != nullptr && a.cls_index[b] == v) ? 1.f : 0.f;
}

}  // namespace fcn

using namespace fcn;

extern "C" int fcn_build_inputs(const fcn_input_args *args, fcn_stream_t stream) {
    FCN_REQUIRE(args != nullptr, "args is NULL");
    const fcn_input_args &a = *args;
    FCN_REQUIRE(a.B >= 0 && a.N >= 1 && a.num_scales >= 0 && a.num_scales <= FCN_MAX_SCALES, "bad sizes");
    if (a.B == 0) return FCN_OK;
    FCN_REQUIRE(a.points && a.point_offsets && a.choice && a.frustum_angle && a.box2d && a.P && a.point_cloud,
                "NULL pointer");
    for (int s = 0; s < a.num_scales; ++s) FCN_REQUIRE(a.centers[s] && a.T[s] >= 1 && a.stride[s] > 0, "bad scale");
    build_inputs_kernel<<<a.B, 256, 0, (cudaStream_t)stream>>>(a);
    FCN_LAUNCH_CHECK();
    return FCN_OK;
}
