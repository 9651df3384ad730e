// gcd_b200 — the non-GEMM kernels of the LPIPS perceptual metric (gcd-model/sgm/modules/autoencoding/lpips/loss/lpips.py,
// VGG16 variant; DiffusionEngine.validation_step, gcd-model/sgm/models/diffusion.py:317-362). The 13 VGG16 convolutions run on
// tc_gemm with the ReLU epilogue (act 3); what is left is
//   - the input stage: ScalingLayer (x - shift) / scale and the 3x3 im2col of conv1_1 (K = 27 taps padded to 64 columns), so that
//     conv1_1 is one K = 64 GEMM instead of a 9-tap conv over 3 channels padded to 64;
//   - MaxPool2d(2, 2), floor mode, on channels-last 16-bit activations;
//   - the head of one tapped layer: per pixel of each (input, target) pair, both features normalised over channels, the squared
//     difference dotted with the layer's `lin` weights, and the spatial mean. The reduction order is fixed (no order-dependent
//     atomics), so the same inputs give the same bits.
#include "common.cuh"
#include "../../include/gcd_b200.h"
#include <atomic>
extern std::atomic<int64_t> g_launches;

namespace {
constexpr int IN_THREADS = 256;
constexpr int HEAD_THREADS = 256;

// one thread per (output pixel, group of 8 columns), so that a warp's 16-byte stores are contiguous. Column j < 27 is tap
// (ky, kx) = ((j / 3) / 3, (j / 3) % 3), channel j % 3 of the scaled image, zero outside the image (the reference zero-pads the
// scaled tensor); columns 27..63 are zero.
__global__ void __launch_bounds__(IN_THREADS)
lpips_input_kernel(const float* __restrict__ in, int n, int H, int W, const float* __restrict__ shift, const float* __restrict__ scale,
                   uint4* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * IN_THREADS + threadIdx.x;
    const int64_t HW = (int64_t)H * W;
    if (i >= n * HW * 8) return;
    const int q = (int)(i & 7);
    if (q >= 4) { out[i] = make_uint4(0u, 0u, 0u, 0u); return; }
    const int64_t r = i >> 3;
    const int f = (int)(r / HW), rem = (int)(r - f * HW), y = rem / W, x = rem - y * W;
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const int j = 8 * q + k, t = j / 3, c = j - 3 * t;
        const int yy = y + t / 3 - 1, xx = x + t % 3 - 1;
        v[k] = (j < 27 && yy >= 0 && yy < H && xx >= 0 && xx < W)
                   ? (__ldg(in + ((int64_t)f * 3 + c) * HW + (int64_t)yy * W + xx) - __ldg(shift + c)) / __ldg(scale + c)
                   : 0.f;
    }
    out[i] = make_uint4(pack2(v[0], v[1]), pack2(v[2], v[3]), pack2(v[4], v[5]), pack2(v[6], v[7]));
}

__device__ __forceinline__ uint32_t max2(uint32_t a, uint32_t b) {
    const float2 x = unpack2(a), y = unpack2(b);
    return pack2(fmaxf(x.x, y.x), fmaxf(x.y, y.y));   // exact: the max of two 16-bit values is one of them
}

// one thread per (output pixel, 8 channels)
__global__ void __launch_bounds__(256)
maxpool2x2_kernel(const uint4* __restrict__ in, int n, int H, int W, int C8, uint4* __restrict__ out) {
    const int Ho = H / 2, Wo = W / 2;
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= (int64_t)n * Ho * Wo * C8) return;
    const int c = (int)(i % C8);
    const int64_t p = i / C8;
    const int x = (int)(p % Wo), y = (int)((p / Wo) % Ho), f = (int)(p / ((int64_t)Wo * Ho));
    const uint4* a = in + (((int64_t)f * H + 2 * y) * W + 2 * x) * C8 + c;
    const uint4 v00 = __ldg(a), v01 = __ldg(a + C8), v10 = __ldg(a + (int64_t)W * C8), v11 = __ldg(a + (int64_t)W * C8 + C8);
    uint4 m;
    m.x = max2(max2(v00.x, v01.x), max2(v10.x, v11.x));
    m.y = max2(max2(v00.y, v01.y), max2(v10.y, v11.y));
    m.z = max2(max2(v00.z, v01.z), max2(v10.z, v11.z));
    m.w = max2(max2(v00.w, v01.w), max2(v10.w, v11.w));
    out[i] = m;
}

// LPIPS head of one tapped layer with C channels. Block (b, pair) reduces pixels [b * GCD_LPIPS_HEAD_PIX, +GCD_LPIPS_HEAD_PIX) of
// the pair to one float64 partial; the last block of a pair to finish (a per-pair counter) sums the pair's partials in block
// order and writes the mean. A group of G lanes works on one pixel at a time, each lane on V vectors of 8 channels.
template <int C>
__global__ void __launch_bounds__(HEAD_THREADS)
lpips_head_kernel(const uint4* __restrict__ feat, int HW, const int32_t* __restrict__ pairs, const float* __restrict__ w,
                  double* __restrict__ partial, uint32_t* __restrict__ count, double* __restrict__ out) {
    constexpr int G = C / 8 < 32 ? C / 8 : 32, V = C / (8 * G), GROUPS = HEAD_THREADS / G;
    constexpr int ITERS = GCD_LPIPS_HEAD_PIX / GROUPS;
    static_assert(GCD_LPIPS_HEAD_PIX % GROUPS == 0, "pixels per block");
    __shared__ double sred[GROUPS];
    __shared__ bool last;
    const int pair = blockIdx.y, nblk = gridDim.x;
    const int g = threadIdx.x / G, l = threadIdx.x % G;
    const uint4* fa = feat + (int64_t)__ldg(pairs + 2 * pair) * HW * (C / 8);
    const uint4* fb = feat + (int64_t)__ldg(pairs + 2 * pair + 1) * HW * (C / 8);
    float wv[8 * V];
#pragma unroll
    for (int v = 0; v < V; v++)
#pragma unroll
        for (int k = 0; k < 8; k++) wv[8 * v + k] = __ldg(w + (v * G + l) * 8 + k);
    double acc = 0.0;
    const int p0 = blockIdx.x * GCD_LPIPS_HEAD_PIX;
    for (int it = 0; it < ITERS; it++) {                      // the same trip count for every lane (shuffles below)
        const int pix = p0 + it * GROUPS + g;
        const bool ok = pix < HW;
        float a[8 * V], b[8 * V];
#pragma unroll
        for (int v = 0; v < V; v++) {
            uint4 qa = make_uint4(0u, 0u, 0u, 0u), qb = qa;
            if (ok) { qa = __ldg(fa + (int64_t)pix * (C / 8) + v * G + l); qb = __ldg(fb + (int64_t)pix * (C / 8) + v * G + l); }
            const uint32_t wa[4] = {qa.x, qa.y, qa.z, qa.w}, wb[4] = {qb.x, qb.y, qb.z, qb.w};
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const float2 ua = unpack2(wa[k]), ub = unpack2(wb[k]);
                a[8 * v + 2 * k] = ua.x; a[8 * v + 2 * k + 1] = ua.y;
                b[8 * v + 2 * k] = ub.x; b[8 * v + 2 * k + 1] = ub.y;
            }
        }
        float sa = 0.f, sb = 0.f;
#pragma unroll
        for (int k = 0; k < 8 * V; k++) { sa += a[k] * a[k]; sb += b[k] * b[k]; }
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) { sa += __shfl_xor_sync(0xffffffffu, sa, o); sb += __shfl_xor_sync(0xffffffffu, sb, o); }
        const float na = sqrtf(sa) + 1e-10f, nb = sqrtf(sb) + 1e-10f;   // normalize_tensor: x / (sqrt(sum x^2) + eps)
        float d = 0.f;
#pragma unroll
        for (int k = 0; k < 8 * V; k++) {
            const float t = a[k] / na - b[k] / nb;
            d += wv[k] * (t * t);
        }
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
        if (ok) acc += (double)d;
    }
    if (l == 0) sred[g] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < GROUPS; i++) s += sred[i];
        partial[(int64_t)pair * nblk + blockIdx.x] = s;
        __threadfence();
        last = atomicAdd(count + pair, 1u) == (unsigned)(nblk - 1);
    }
    __syncthreads();
    if (!last) return;
    // last block of the pair: the partials of all its blocks are visible (each was fenced before its block's count)
    __threadfence();
    double s = 0.0;
    for (int i = threadIdx.x; i < nblk; i += HEAD_THREADS) s += __ldcg(partial + (int64_t)pair * nblk + i);
    __shared__ double sfin[HEAD_THREADS];
    sfin[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < HEAD_THREADS; i++) t += sfin[i];
        out[pair] = t / (double)HW;
        count[pair] = 0u;                                       // ready for the next launch
    }
}
}  // namespace

extern "C" int gcd_lpips_input(const float* in, int n, int H, int W, const float* shift, const float* scale, void* out, void* stream) {
    GCD_REQUIRE(in && shift && scale && out && n > 0 && H > 0 && W > 0, "lpips_input: bad arguments");
    GCD_REQUIRE(((uintptr_t)out & 15) == 0, "lpips_input: out must be 16-byte aligned");
    const int64_t threads = (int64_t)n * H * W * 8;
    lpips_input_kernel<<<(unsigned)((threads + IN_THREADS - 1) / IN_THREADS), IN_THREADS, 0, (cudaStream_t)stream>>>(
        in, n, H, W, shift, scale, reinterpret_cast<uint4*>(out));
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches++;
    return 0;
}

extern "C" int gcd_maxpool2x2(const void* in, int n, int H, int W, int C, void* out, void* stream) {
    GCD_REQUIRE(in && out && n > 0 && H >= 2 && W >= 2 && C > 0 && C % 8 == 0, "maxpool2x2: need [n, H >= 2, W >= 2, C %% 8 == 0]");
    GCD_REQUIRE(((uintptr_t)in & 15) == 0 && ((uintptr_t)out & 15) == 0, "maxpool2x2: tensors must be 16-byte aligned");
    const int64_t total = (int64_t)n * (H / 2) * (W / 2) * (C / 8);
    maxpool2x2_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const uint4*>(in), n, H, W,
                                                                                         C / 8, reinterpret_cast<uint4*>(out));
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches++;
    return 0;
}

extern "C" int gcd_lpips_head(const void* feat, int HW, int C, const int32_t* pairs, int n_pairs, const float* w, double* partial,
                              uint32_t* count, double* out, void* stream) {
    GCD_REQUIRE(feat && pairs && w && partial && count && out && HW > 0 && n_pairs > 0 && n_pairs <= 65535,
                "lpips_head: bad arguments");
    GCD_REQUIRE(((uintptr_t)feat & 15) == 0 && ((uintptr_t)w & 15) == 0, "lpips_head: feat and w must be 16-byte aligned");
    const int nblk = (HW + GCD_LPIPS_HEAD_PIX - 1) / GCD_LPIPS_HEAD_PIX;
    const dim3 grid(nblk, n_pairs);
    const uint4* f = reinterpret_cast<const uint4*>(feat);
    cudaStream_t st = (cudaStream_t)stream;
    switch (C) {
        case 64: lpips_head_kernel<64><<<grid, HEAD_THREADS, 0, st>>>(f, HW, pairs, w, partial, count, out); break;
        case 128: lpips_head_kernel<128><<<grid, HEAD_THREADS, 0, st>>>(f, HW, pairs, w, partial, count, out); break;
        case 256: lpips_head_kernel<256><<<grid, HEAD_THREADS, 0, st>>>(f, HW, pairs, w, partial, count, out); break;
        case 512: lpips_head_kernel<512><<<grid, HEAD_THREADS, 0, st>>>(f, HW, pairs, w, partial, count, out); break;
        default: GCD_REQUIRE(false, "lpips_head: C=%d unsupported (64, 128, 256 or 512)", C);
    }
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches++;
    return 0;
}
