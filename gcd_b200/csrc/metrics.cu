// gcd_b200 — per-frame image metrics of the evaluation loop (SURVEY.md §8(f) rank 3): PSNR and SSIM, full-frame and over a
// mask, of decoded frames against ground truth — gcd-model/scripts/test.py:346-496 (calculate_metrics), whose SSIM is
// scikit-image 0.22.0 `structural_similarity(data_range=1, channel_axis=0)` and gcd-model/scripts/eval_utils.py:571-664
// (masked_ssim: the same map averaged over an eroded mask): 7x7 uniform window, sample covariance (NP/(NP-1)), K1 = 0.01,
// K2 = 0.03, the 3-pixel border strip ignored, mean over the three channels.
// One block per 32x16 output tile and channel, the 38x22 halo of both images staged in shared memory. The arithmetic follows the
// reference's float32 numpy / scipy arithmetic, because in flat and near-flat windows (sky, floors, 8-bit levels) SSIM is the
// difference of two nearly equal window means over C2 = 9e-4, and any other rounding of those means moves it by up to 1e-3:
//   * products x*x, y*y, x*y rounded to fp32;
//   * window means as scipy.ndimage.uniform_filter forms them: a vertical pass (axis 0) then a horizontal one, each summing its
//     7 fp32 inputs in fp64, dividing by 7 in fp64 and rounding to fp32 once (the vertical means of the tile's 38 halo columns
//     go through a shared-memory table); scipy keeps a running mean instead of a fresh sum, which rarely lands one fp32 ulp away;
//   * the SSIM formula in fp32 in numpy's operation order, every operation rounded on its own (no FMA contraction);
//   * PSNR: the difference squared in fp32 (skimage's mean_squared_error on float32 images), summed in fp64.
// Block reduction in fp64, one fp64 atomic per block and quantity.
#include "common.cuh"
#include "../../include/gcd_b200.h"
#include <atomic>
extern std::atomic<int64_t> g_launches;

namespace {
constexpr int TX = 32, TY = 16, R = 3, HX = TX + 2 * R, HY = TY + 2 * R, NQ = 5;

// s / 7 correctly rounded in fp64 (Markstein: q0 = s * RN(1/7) is within one ulp and the remainder s - 7 q0 is exact), then
// rounded to fp32: one pass of scipy's uniform_filter1d on a float32 array
__device__ __forceinline__ float mean7(double s) {
    const double q0 = __dmul_rn(s, 1.0 / 7.0);
    return __double2float_rn(__fma_rn(__fma_rn(-7.0, q0, s), 1.0 / 7.0, q0));
}

// out per frame: [0] sum sq. diff (all), [1] count, [2] sum sq. diff (mask), [3] count (mask), [4] sum SSIM (cropped map),
// [5] count, [6] sum SSIM over the eroded mask, [7] count  — sums over the 3 channels
__global__ void __launch_bounds__(TX * TY)
frame_metrics_kernel(const float* __restrict__ a, const float* __restrict__ b, const uint8_t* __restrict__ mask, int H, int W,
                     double* __restrict__ out) {
    __shared__ float sa[HY][HX + 1], sb[HY][HX + 1];
    __shared__ uint8_t sm[HY][HX + 1];
    __shared__ double vmean[NQ][TY][HX];       // vertical 7-row means (fp32 values) of x, y, x*x, y*y, x*y per halo column
    __shared__ double red[8][TX * TY / 32];
    const int f = blockIdx.z / 3, c = blockIdx.z % 3;
    const float* pa = a + ((int64_t)f * 3 + c) * H * W;
    const float* pb = b + ((int64_t)f * 3 + c) * H * W;
    const uint8_t* pm = mask ? mask + (int64_t)f * H * W : nullptr;
    const int x0 = blockIdx.x * TX, y0 = blockIdx.y * TY;
    for (int i = threadIdx.x; i < HX * HY; i += TX * TY) {
        const int ly = i / HX, lx = i % HX, y = y0 + ly - R, x = x0 + lx - R;
        const bool in = y >= 0 && y < H && x >= 0 && x < W;
        sa[ly][lx] = in ? pa[(int64_t)y * W + x] : 0.f;
        sb[ly][lx] = in ? pb[(int64_t)y * W + x] : 0.f;
        sm[ly][lx] = (in && pm) ? pm[(int64_t)y * W + x] : 0;      // binary_erosion border_value = 0
    }
    __syncthreads();
    if (threadIdx.x < 2 * NQ * HX) {           // vertical pass: one thread per quantity, halo column and half of the tile's rows
        const int q = threadIdx.x / (2 * HX), lx = threadIdx.x % HX, r0 = (threadIdx.x / HX) % 2 * (TY / 2);
        double v[TY / 2 + 2 * R];
#pragma unroll
        for (int r = 0; r < TY / 2 + 2 * R; r++) {   // quantity q = u * w with u, w in {x, y, 1} (x * 1 is exact)
            const float x = sa[r0 + r][lx], y = sb[r0 + r][lx];
            const float u = (q == 1 || q == 3) ? y : x, w = q < 2 ? 1.f : (q == 2 ? x : y);
            v[r] = (double)__fmul_rn(u, w);
        }
#pragma unroll
        for (int r = 0; r < TY / 2; r++) {
            double s = v[r];
#pragma unroll
            for (int k = 1; k < 7; k++) s += v[r + k];
            vmean[q][r0 + r][lx] = (double)mean7(s);
        }
    }
    __syncthreads();
    const int lx = threadIdx.x % TX, ly = threadIdx.x / TX, x = x0 + lx, y = y0 + ly;
    double v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (x < W && y < H) {
        const float d = __fsub_rn(sa[ly + R][lx + R], sb[ly + R][lx + R]);
        v[0] = (double)__fmul_rn(d, d); v[1] = 1.0;
        if (pm && sm[ly + R][lx + R]) { v[2] = v[0]; v[3] = 1.0; }
        if (x >= R && x < W - R && y >= R && y < H - R) {          // crop(S, pad): windows fully inside the image
            float m[NQ];                                            // ux, uy, uxx, uyy, uxy
#pragma unroll
            for (int q = 0; q < NQ; q++) {                          // horizontal pass over the 7 vertical means
                double s = vmean[q][ly][lx];
#pragma unroll
                for (int k = 1; k < 7; k++) s += vmean[q][ly][lx + k];
                m[q] = mean7(s);
            }
            const float ux = m[0], uy = m[1], uxx = m[2], uyy = m[3], uxy = m[4];
            const float cov = (float)(49.0 / 48.0), C1 = (float)(0.01 * 0.01), C2 = (float)(0.03 * 0.03);
            const float ux2 = __fmul_rn(ux, ux), uy2 = __fmul_rn(uy, uy);
            const float vx = __fmul_rn(cov, __fsub_rn(uxx, ux2)), vy = __fmul_rn(cov, __fsub_rn(uyy, uy2)),
                        vxy = __fmul_rn(cov, __fsub_rn(uxy, __fmul_rn(ux, uy)));
            const float A1 = __fadd_rn(__fmul_rn(__fmul_rn(2.f, ux), uy), C1), A2 = __fadd_rn(__fmul_rn(2.f, vxy), C2);
            const float B1 = __fadd_rn(__fadd_rn(ux2, uy2), C1), B2 = __fadd_rn(__fadd_rn(vx, vy), C2);
            const float S = __fdiv_rn(__fmul_rn(A1, A2), __fmul_rn(B1, B2));
            v[4] = S; v[5] = 1.0;
            if (pm) {          // binary_erosion(mask, iterations = 3) with the cross element = all pixels within L1 distance 3
                bool ok = true;
#pragma unroll
                for (int dy = -R; dy <= R; dy++)
#pragma unroll
                    for (int dx = -R; dx <= R; dx++)
                        if (abs(dx) + abs(dy) <= R) ok = ok && sm[ly + R + dy][lx + R + dx];
                if (ok) { v[6] = S; v[7] = 1.0; }
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 8; k++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
        if ((threadIdx.x & 31) == 0) red[k][threadIdx.x >> 5] = v[k];
    }
    __syncthreads();
    if (threadIdx.x < 8) {
        double s = 0.0;
        for (int w = 0; w < TX * TY / 32; w++) s += red[threadIdx.x][w];
        if (s != 0.0) atomicAdd(out + (int64_t)f * 8 + threadIdx.x, s);
    }
}
}  // namespace

extern "C" int gcd_frame_metrics(const float* pred, const float* gt, const uint8_t* mask, int frames, int H, int W, double* out,
                                 void* stream) {
    GCD_REQUIRE(pred && gt && out && frames > 0 && H >= 7 && W >= 7, "frame_metrics: need [frames, 3, H >= 7, W >= 7] images");
    GCD_REQUIRE((int64_t)frames * 3 <= 65535, "frame_metrics: too many frames for one launch");
    cudaStream_t st = (cudaStream_t)stream;
    GCD_CUDA_CHECK(cudaMemsetAsync(out, 0, (size_t)frames * 8 * sizeof(double), st));
    dim3 grid((W + TX - 1) / TX, (H + TY - 1) / TY, frames * 3);
    frame_metrics_kernel<<<grid, TX * TY, 0, st>>>(pred, gt, mask, H, W, out);
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches++;
    return 0;
}
