// gcd_b200 — the OpenCLIP ViT-H/14 image tower of the GCD conditioner (encoders/modules.py:653-815, open_clip 2.23.0
// VisionTransformer): the input preprocessing + patch unfold, and self-attention with head_dim 80. The GEMMs (patch
// embedding, QKV, out_proj, MLP, proj) run on gemm.cu's tc_gemm and the LayerNorms on norm.cu.
#include "common.cuh"
#include "../../include/gcd_b200.h"
#include <atomic>
extern std::atomic<int64_t> g_launches;

// ---------------------------------------------------------------------------------------------- preprocessing
// kornia 0.7.0 resize(antialias=True): separable Gaussian blur, horizontal pass first, PyTorch 'reflect' border (the edge
// pixel is not repeated). One thread per output pixel of one channel plane; taps come from the host.
__device__ __forceinline__ int reflect_idx(int i, int n) {
    if (n == 1) return 0;
    while (i < 0 || i >= n) i = i < 0 ? -i : 2 * (n - 1) - i;
    return i;
}

template <bool HORIZ>
__global__ void clip_blur_kernel(const float* __restrict__ in, int planes, int H, int W, const float* __restrict__ taps,
                                 int ks, float* __restrict__ out) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = (int64_t)planes * H * W;
    if (idx >= total) return;
    const int x = (int)(idx % W);
    const int y = (int)((idx / W) % H);
    const float* src = in + (idx / ((int64_t)H * W)) * H * W;
    const int r = ks / 2;
    float acc = 0.f;
    for (int t = 0; t < ks; t++) {
        const float w = __ldg(taps + t);
        acc += HORIZ ? w * src[(int64_t)y * W + reflect_idx(x + t - r, W)] : w * src[(int64_t)reflect_idx(y + t - r, H) * W + x];
    }
    out[idx] = acc;
}

// PyTorch upsample_bicubic2d (align_corners=True): cubic convolution with A = -0.75, source taps clamped to the border.
__device__ __forceinline__ float cubic1(float x) { return ((-0.75f + 2.0f) * x - (-0.75f + 3.0f)) * x * x + 1.0f; }
__device__ __forceinline__ float cubic2(float x) { return ((-0.75f * x - 5.0f * -0.75f) * x + 8.0f * -0.75f) * x - 4.0f * -0.75f; }
__device__ __forceinline__ void cubic_coeffs(float t, float (&c)[4]) {
    c[0] = cubic2(t + 1.0f);
    c[1] = cubic1(t);
    c[2] = cubic1(1.0f - t);
    c[3] = cubic2(2.0f - t);
}

// One thread per element of the patch matrix [n*257, 640]: row 0 of an image (class-token slot) and columns >= 588 are
// zero; row 1 + py*16 + px, column (ky*14 + kx)*3 + c holds normalised pixel (py*14 + ky, px*14 + kx) of channel c.
template <typename OutT>   // act_t for the patch-embedding GEMM; float to check the preprocessing itself
__global__ void clip_patchify_kernel(const float* __restrict__ img, int n, int H, int W, int resize, float sy, float sx,
                                     const float* __restrict__ mean_std, OutT* __restrict__ out) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = (int64_t)n * 257 * 640;
    if (idx >= total) return;
    const int col = (int)(idx % 640);
    const int64_t row = idx / 640;
    const int tok = (int)(row % 257);
    const int b = (int)(row / 257);
    if (tok == 0 || col >= 588) { out[idx] = OutT(0.f); return; }
    const int p = tok - 1, py = p >> 4, px = p & 15;
    const int c = col % 3, kx = (col / 3) % 14, ky = col / 42;
    const int oy = py * 14 + ky, ox = px * 14 + kx;
    const float* src = img + ((int64_t)b * 3 + c) * H * W;
    float v;
    if (!resize) {
        v = src[(int64_t)oy * W + ox];
    } else {
        const float ry = sy * (float)oy, rx = sx * (float)ox;
        const int iy = (int)floorf(ry), ix = (int)floorf(rx);
        float cy[4], cx[4];
        cubic_coeffs(ry - (float)iy, cy);
        cubic_coeffs(rx - (float)ix, cx);
        v = 0.f;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int yy = min(max(iy - 1 + j, 0), H - 1);
            float rowv = 0.f;
#pragma unroll
            for (int i = 0; i < 4; i++) rowv += cx[i] * src[(int64_t)yy * W + min(max(ix - 1 + i, 0), W - 1)];
            v += cy[j] * rowv;
        }
    }
    v = (v + 1.0f) / 2.0f;
    v = (v - __ldg(mean_std + c)) / __ldg(mean_std + 3 + c);
    if constexpr (sizeof(OutT) == 4) out[idx] = v;
    else out[idx] = f2act(v);
}

extern "C" int gcd_clip_preprocess(const float* in, int n, int H, int W, const float* taps_x, int ks_x, const float* taps_y,
                                   int ks_y, float* scratch, const float* mean_std, void* out, int out_f32, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GCD_REQUIRE(in && mean_std && out && n > 0 && H > 0 && W > 0, "clip_preprocess: bad arguments");
    const bool blur = ks_x > 0;
    GCD_REQUIRE(!blur || (taps_x && taps_y && ks_y > 0 && (ks_x & 1) && (ks_y & 1) && scratch),
                "clip_preprocess: the blur needs odd tap counts and a scratch buffer of 2*n*3*H*W floats");
    const int resize = !(H == 224 && W == 224);
    GCD_REQUIRE(resize || !blur, "clip_preprocess: a 224x224 input passes through unchanged (no blur)");
    const int64_t plane_elems = (int64_t)n * 3 * H * W;
    const float* img = in;
    if (blur) {
        const unsigned blocks = (unsigned)((plane_elems + 255) / 256);
        clip_blur_kernel<true><<<blocks, 256, 0, st>>>(in, n * 3, H, W, taps_x, ks_x, scratch);
        GCD_CUDA_CHECK(cudaGetLastError());
        clip_blur_kernel<false><<<blocks, 256, 0, st>>>(scratch, n * 3, H, W, taps_y, ks_y, scratch + plane_elems);
        GCD_CUDA_CHECK(cudaGetLastError());
        g_launches += 2;
        img = scratch + plane_elems;
    }
    // area_pixel_compute_scale(align_corners=True) = (in - 1) / (out - 1)
    const float sy = (float)(H - 1) / 223.0f, sx = (float)(W - 1) / 223.0f;
    const int64_t total = (int64_t)n * 257 * 640;
    const unsigned blocks = (unsigned)((total + 255) / 256);
    if (out_f32) clip_patchify_kernel<float><<<blocks, 256, 0, st>>>(img, n, H, W, resize, sy, sx, mean_std, (float*)out);
    else clip_patchify_kernel<act_t><<<blocks, 256, 0, st>>>(img, n, H, W, resize, sy, sx, mean_std, (act_t*)out);
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches++;
    return 0;
}

// ---------------------------------------------------------------------------------------------- attention, head_dim 80
// nn.MultiheadAttention self-attention of the ViT (16 heads x 80, L = 257 tokens). One CTA of 4 warps per (image, head,
// 64-query block); each warp owns 16 query rows with Q fragments in registers. K/V are streamed in 64-key blocks through
// shared memory and consumed by mma.sync m16n8k16 (d = 80 is five k-steps of 16; wgmma's M = 64 per warpgroup would pad
// the 257-token sequence the same way but needs the 128B-swizzled layout, which 160-byte rows do not fit). Online softmax in
// fp32 (FlashAttention-2), P re-packed in registers as the A operand of P.V; scores never leave the SM.
namespace {
constexpr int D80 = 80;
constexpr int AP = 88;    // halves per staged row: 176 B, eight consecutive rows hit distinct 16-byte bank groups (ldmatrix)
constexpr int QB = 64;    // queries per CTA
constexpr int KB = 64;    // keys per block

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(ptx::smem_u32(p)));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(ptx::smem_u32(p)));
}
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
#ifdef GCD_ACT_BF16
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
#else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
#endif
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
}  // namespace

__global__ void __launch_bounds__(128)
attn_d80_kernel(const act_t* __restrict__ qkv, int L, int heads, float scale_log2, act_t* __restrict__ out) {
    __shared__ __align__(16) act_t sq[QB][AP];
    __shared__ __align__(16) act_t sk[KB][AP];
    __shared__ __align__(16) act_t sv[KB][AP];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * QB, h = blockIdx.y, b = blockIdx.z;
    const int C = heads * D80;
    const int64_t ld = 3 * (int64_t)C;
    const act_t* base = qkv + (int64_t)b * L * ld + h * D80;
    const uint4 zero = make_uint4(0, 0, 0, 0);

    // ---- stage Q (64 rows x 10 chunks of 16 B; rows past L read as zero)
    for (int i = threadIdx.x; i < QB * 10; i += 128) {
        const int r = i / 10, ch = i % 10;
        *reinterpret_cast<uint4*>(&sq[r][ch * 8]) =
            q0 + r < L ? *reinterpret_cast<const uint4*>(base + (int64_t)(q0 + r) * ld + ch * 8) : zero;
    }
    __syncthreads();
    uint32_t qa[5][4];
#pragma unroll
    for (int kk = 0; kk < 5; kk++) ldsm_x4(qa[kk], &sq[warp * 16 + (lane & 15)][kk * 16 + (lane >> 4) * 8]);

    float o[10][4];
#pragma unroll
    for (int i = 0; i < 10; i++) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    const int t2 = (lane & 3) * 2;

    for (int k0 = 0; k0 < L; k0 += KB) {
        __syncthreads();                                    // the previous block's K/V have been consumed
        for (int i = threadIdx.x; i < KB * 20; i += 128) {
            const int r = (i >> 1) / 10, ch = (i >> 1) % 10, which = i & 1;
            const bool ok = k0 + r < L;
            const act_t* src = base + (int64_t)(k0 + r) * ld + (which + 1) * C + ch * 8;
            uint4 v = ok ? *reinterpret_cast<const uint4*>(src) : zero;
            *reinterpret_cast<uint4*>(which ? &sv[r][ch * 8] : &sk[r][ch * 8]) = v;
        }
        __syncthreads();
        // ---- S = Q K^T: 16 x 64 per warp
        float s[8][4];
#pragma unroll
        for (int j = 0; j < 8; j++) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
        for (int kk = 0; kk < 5; kk++) {
#pragma unroll
            for (int nb = 0; nb < 4; nb++) {
                uint32_t bk[4];
                ldsm_x4(bk, &sk[nb * 16 + (lane & 7) + ((lane >> 4) << 3)][kk * 16 + ((lane >> 3) & 1) * 8]);
                mma16816(s[2 * nb], qa[kk], bk[0], bk[1]);
                mma16816(s[2 * nb + 1], qa[kk], bk[2], bk[3]);
            }
        }
        // ---- online softmax (log2 domain); rows g (elements 0,1) and g + 8 (elements 2,3)
        float bm0 = -INFINITY, bm1 = -INFINITY;
#pragma unroll
        for (int j = 0; j < 8; j++) {
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const bool ok = k0 + j * 8 + t2 + e < L;
                s[j][e] = ok ? s[j][e] * scale_log2 : -INFINITY;
                s[j][2 + e] = ok ? s[j][2 + e] * scale_log2 : -INFINITY;
                bm0 = fmaxf(bm0, s[j][e]);
                bm1 = fmaxf(bm1, s[j][2 + e]);
            }
        }
        bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 1)); bm0 = fmaxf(bm0, __shfl_xor_sync(0xffffffffu, bm0, 2));
        bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 1)); bm1 = fmaxf(bm1, __shfl_xor_sync(0xffffffffu, bm1, 2));
        const float nm0 = fmaxf(m0, bm0), nm1 = fmaxf(m1, bm1);   // finite: every key block holds at least one valid key
        const float al0 = exp2f(m0 - nm0), al1 = exp2f(m1 - nm1);
        m0 = nm0; m1 = nm1;
        l0 *= al0; l1 *= al1;
#pragma unroll
        for (int i = 0; i < 10; i++) { o[i][0] *= al0; o[i][1] *= al0; o[i][2] *= al1; o[i][3] *= al1; }
        // P = 2^15 exp2(s - m) (largest 32768): the offset keeps weights down to 2^-40 of the row maximum out of fp16's
        // flush-to-zero range when P is packed for P.V; l carries the same power of two
        const float ms0 = m0 - 15.f, ms1 = m1 - 15.f;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            s[j][0] = exp2f(s[j][0] - ms0); s[j][1] = exp2f(s[j][1] - ms0);
            s[j][2] = exp2f(s[j][2] - ms1); s[j][3] = exp2f(s[j][3] - ms1);
            l0 += s[j][0] + s[j][1];
            l1 += s[j][2] + s[j][3];
        }
        // ---- O += P V: four k-steps of 16 keys, ten 8-column tiles of d
#pragma unroll
        for (int kk = 0; kk < 4; kk++) {
            const uint32_t pa[4] = {pack2(s[2 * kk][0], s[2 * kk][1]), pack2(s[2 * kk][2], s[2 * kk][3]),
                                    pack2(s[2 * kk + 1][0], s[2 * kk + 1][1]), pack2(s[2 * kk + 1][2], s[2 * kk + 1][3])};
#pragma unroll
            for (int d0 = 0; d0 < D80; d0 += 16) {
                uint32_t bv[4];
                ldsm_x4_t(bv, &sv[kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8][d0 + (lane >> 4) * 8]);
                mma16816(o[d0 / 8], pa, bv[0], bv[1]);
                mma16816(o[d0 / 8 + 1], pa, bv[2], bv[3]);
            }
        }
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
    const int r0 = q0 + warp * 16 + (lane >> 2), r1 = r0 + 8;
    act_t* ob = out + (int64_t)b * L * C + h * D80;
#pragma unroll
    for (int i = 0; i < 10; i++) {
        if (r0 < L) *reinterpret_cast<uint32_t*>(ob + (int64_t)r0 * C + i * 8 + t2) = pack2(o[i][0] * inv0, o[i][1] * inv0);
        if (r1 < L) *reinterpret_cast<uint32_t*>(ob + (int64_t)r1 * C + i * 8 + t2) = pack2(o[i][2] * inv1, o[i][3] * inv1);
    }
}

extern "C" int gcd_attention_d80(const void* qkv, int n, int L, int heads, void* out, void* stream) {
    GCD_REQUIRE(qkv && out && n > 0 && heads > 0, "attention_d80: bad arguments");
    GCD_REQUIRE(L >= 1 && L <= 1024, "attention_d80: L=%d unsupported (1..1024)", L);
    GCD_REQUIRE(((uintptr_t)qkv & 15) == 0 && ((uintptr_t)out & 15) == 0, "attention_d80: tensors must be 16B aligned");
    GCD_REQUIRE(n <= 65535 && heads <= 65535, "attention_d80: too many images or heads");
    const float scale_log2 = 1.4426950408889634f / sqrtf((float)D80);
    dim3 grid((L + QB - 1) / QB, heads, n);
    attn_d80_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>((const act_t*)qkv, L, heads, scale_log2, (act_t*)out);
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches++;
    return 0;
}
