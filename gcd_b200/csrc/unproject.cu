// gcd_b200 — RGB-D to point-cloud unprojection of the dataset conversion (data-gen/data_utils.py:91-138 unproject_pixels_to_points
// and camera_to_world, with convert_pcl_kubric.py:96-121 correct_depth_ball_plane_torch or convert_pcl_pardom.py:166's clamp).
// One thread per pixel, all (frame, view) images of a group in one launch; writes the stored fp16 xyz [n, H*W, 3].
//
// The arithmetic restates the reference's float32 torch ops on CUDA: every product, sum and quotient is its own fp32 rounding
// (__fmul_rn / __fadd_rn / __fdiv_rn, no FMA contraction), atanf / tanf / sqrtf are libdevice's, as torch's unary CUDA ops.
//   ball -> plane (Kubric): fov = 2 * atan(rcp(2 |fx|) * W) (torch's `W / t` is `t.reciprocal() * W`), linspace(-fov/2, fov/2, W)
//     with torch's two-sided formula, correction = sqrt((tan(ax)^2 + tan(ay)^2) + 1), z = depth / correction;
//   clamp (ParDom): z = min(max(depth, 0), max_depth), NaN kept (torch.clamp);
//   x = ((u - cx) * z) / fx, y = ((v - cy) * z) / fy;
//   world_i = ((R_i0 x + R_i1 y) + R_i2 z) + t_i  — this summation order; torch's `xyz @ R.T` is a BLAS product whose order is
//     the library's, so the stored fp16 can differ from a reference run by one ulp where the fp32 sums round differently;
//   stored with round-to-nearest-even (__float2half_rn: overflow gives +-inf, as `.half()`).
#include "common.cuh"
#include "../../include/gcd_b200.h"
#include <atomic>
#include <math.h>
extern std::atomic<int64_t> g_launches;

namespace {
constexpr int UT = 128;

// torch.linspace(start, end, steps)[i] in fp32 (aten RangeFactories.cu): step = (end - start) / (steps - 1),
// start + step * i below steps / 2, end - step * (steps - 1 - i) from there on.
__device__ __forceinline__ float linspace_at(float start, float end, int steps, int i) {
    if (steps == 1) return start;
    const float step = __fdiv_rn(__fsub_rn(end, start), (float)(steps - 1));
    if (i < steps / 2) return __fadd_rn(start, __fmul_rn(step, (float)i));
    return __fsub_rn(end, __fmul_rn(step, (float)(steps - 1 - i)));
}

// tan of the view angle of index i of n pixels along an axis with focal length f (correct_depth_ball_plane_torch)
__device__ __forceinline__ float ball_tan(float f, int n, int i) {
    const float rcp = __fdiv_rn(1.f, __fmul_rn(2.f, fabsf(f)));
    const float fov = __fmul_rn(2.f, atanf(__fmul_rn(rcp, (float)n)));
    const float half = __fmul_rn(fov, 0.5f);
    return tanf(linspace_at(-half, half, n, i));
}

__global__ void __launch_bounds__(UT) unproject_kernel(const float* __restrict__ depth, int H, int W,
                                                       const float* __restrict__ cams, int mode, float max_depth,
                                                       __half* __restrict__ out) {
    const int u = blockIdx.x * UT + threadIdx.x;
    if (u >= W) return;
    const int v = blockIdx.y, img = blockIdx.z;
    const float* c = cams + (int64_t)img * GCD_UNPROJECT_CAM;
    const float fx = c[0], fy = c[1], cx = c[2], cy = c[3];
    const int64_t pix = ((int64_t)img * H + v) * W + u;
    float z = depth[pix];
    if (mode == GCD_UNPROJECT_BALL_TO_PLANE) {
        const float mx = ball_tan(fx, W, u), my = ball_tan(fy, H, v);
        const float corr = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(mx, mx), __fmul_rn(my, my)), 1.f));
        z = __fdiv_rn(z, corr);
    } else if (!isnan(z)) {
        z = fminf(fmaxf(z, 0.f), max_depth);
    }
    const float x = __fdiv_rn(__fmul_rn(__fsub_rn((float)u, cx), z), fx);
    const float y = __fdiv_rn(__fmul_rn(__fsub_rn((float)v, cy), z), fy);
    __half* o = out + pix * 3;
#pragma unroll
    for (int i = 0; i < 3; i++) {
        const float* R = c + 4 + 3 * i;
        const float w = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(R[0], x), __fmul_rn(R[1], y)), __fmul_rn(R[2], z)), c[13 + i]);
        o[i] = __float2half_rn(w);
    }
}
}  // namespace

extern "C" int gcd_unproject_depth(const float* depth, int n, int H, int W, const float* cams, int mode, float max_depth, void* out,
                                   void* stream) {
    GCD_REQUIRE(depth && cams && out, "unproject_depth: null pointer");
    GCD_REQUIRE(n > 0 && n <= 65535 && H > 0 && H <= 65535 && W > 0, "unproject_depth: bad sizes n %d, H %d, W %d (n, H <= 65535)",
                n, H, W);
    GCD_REQUIRE(mode == GCD_UNPROJECT_CLAMP || mode == GCD_UNPROJECT_BALL_TO_PLANE, "unproject_depth: unknown mode %d", mode);
    const dim3 grid((unsigned)((W + UT - 1) / UT), H, n);
    unproject_kernel<<<grid, UT, 0, (cudaStream_t)stream>>>(depth, H, W, cams, mode, max_depth, (__half*)out);
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches += 1;
    return 0;
}
