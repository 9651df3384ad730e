// gcd_b200 — temporal self-attention over the T (=14) frames of a clip, per (spatial position, head), head_dim 64.
// Reference: gcd-model/sgm/modules/video_attention.py:109-140 (VideoTransformerBlock.attn1 after the
// "(b t) s c -> (b s) t c" rearrange) with CrossAttention math attention.py:255-344: softmax(q k^T / sqrt(64)) v.
// The rearrange is pure indexing here: tokens stay in [clip, t, s, C] order.
// Work is 0.04 TFLOP per UNet forward: CUDA-core kernel, one thread per (clip, s, head, query frame); the 14 threads of
// a (s, head) group read the same K/V rows (warp-broadcast loads). HBM-bound: reads qkv once, writes out once.
#include "common.cuh"
#include "../../include/gcd_b200.h"
#include <atomic>
extern std::atomic<int64_t> g_launches;

template <int GS>  // lanes per (s, head) group: 16 (T <= 16) or 32
__global__ void __launch_bounds__(128)
attn_temporal_kernel(const act_t* __restrict__ qkv, int clips, int T, int tokens, int heads, act_t* __restrict__ out) {
    const int C = heads * 64;
    const int64_t gid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / GS;   // (clip, s, head)
    const int t = threadIdx.x % GS;
    const int64_t ngroups = (int64_t)clips * tokens * heads;
    if (gid >= ngroups || t >= T) return;
    const int h = (int)(gid % heads);
    const int64_t cs = gid / heads;
    const int s = (int)(cs % tokens);
    const int b = (int)(cs / tokens);
    const int64_t frame_stride = (int64_t)tokens * 3 * C;                       // elements between frames
    const act_t* base = qkv + ((int64_t)b * T * tokens + s) * 3 * C + h * 64;   // frame 0 of this (b, s, head)

    float q[64];
    {
        const uint4* qp = reinterpret_cast<const uint4*>(base + (int64_t)t * frame_stride);
#pragma unroll
        for (int i = 0; i < 8; i++) {
            uint4 v = qp[i];
            float2 f;
            f = unpack2(v.x); q[i * 8 + 0] = f.x; q[i * 8 + 1] = f.y;
            f = unpack2(v.y); q[i * 8 + 2] = f.x; q[i * 8 + 3] = f.y;
            f = unpack2(v.z); q[i * 8 + 4] = f.x; q[i * 8 + 5] = f.y;
            f = unpack2(v.w); q[i * 8 + 6] = f.x; q[i * 8 + 7] = f.y;
        }
    }
    float sc[32];
    float m = -INFINITY;
    for (int j = 0; j < T; j++) {
        const uint4* kp = reinterpret_cast<const uint4*>(base + (int64_t)j * frame_stride + C);
        float acc = 0.f;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            uint4 v = kp[i];
            float2 f;
            f = unpack2(v.x); acc += q[i * 8 + 0] * f.x + q[i * 8 + 1] * f.y;
            f = unpack2(v.y); acc += q[i * 8 + 2] * f.x + q[i * 8 + 3] * f.y;
            f = unpack2(v.z); acc += q[i * 8 + 4] * f.x + q[i * 8 + 5] * f.y;
            f = unpack2(v.w); acc += q[i * 8 + 6] * f.x + q[i * 8 + 7] * f.y;
        }
        acc *= 0.125f;
        sc[j] = acc;
        m = fmaxf(m, acc);
    }
    float l = 0.f;
    for (int j = 0; j < T; j++) { sc[j] = __expf(sc[j] - m); l += sc[j]; }
    const float inv = 1.0f / l;
    float o[64];
#pragma unroll
    for (int i = 0; i < 64; i++) o[i] = 0.f;
    for (int j = 0; j < T; j++) {
        const uint4* vp = reinterpret_cast<const uint4*>(base + (int64_t)j * frame_stride + 2 * C);
        const float pj = sc[j] * inv;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            uint4 v = vp[i];
            float2 f;
            f = unpack2(v.x); o[i * 8 + 0] += pj * f.x; o[i * 8 + 1] += pj * f.y;
            f = unpack2(v.y); o[i * 8 + 2] += pj * f.x; o[i * 8 + 3] += pj * f.y;
            f = unpack2(v.z); o[i * 8 + 4] += pj * f.x; o[i * 8 + 5] += pj * f.y;
            f = unpack2(v.w); o[i * 8 + 6] += pj * f.x; o[i * 8 + 7] += pj * f.y;
        }
    }
    uint4* op = reinterpret_cast<uint4*>(out + (((int64_t)b * T + t) * tokens + s) * C + h * 64);
#pragma unroll
    for (int i = 0; i < 8; i++)
        op[i] = make_uint4(pack2(o[i * 8 + 0], o[i * 8 + 1]), pack2(o[i * 8 + 2], o[i * 8 + 3]),
                           pack2(o[i * 8 + 4], o[i * 8 + 5]), pack2(o[i * 8 + 6], o[i * 8 + 7]));
}

// ---------------------------------------------------------------------------------------------------------------------
// T <= 16: one warp per (clip, position, head) on the legacy warp-level tensor path (mma.sync m16n8k16; a 14x14 problem
// is far below wgmma's M=64 minimum). Q/K/V rows are staged with coalesced 16-byte loads, fragments come from
// ldmatrix, P is reused in registers as the A operand of P.V (FlashAttention-2 layout identity). HBM-bound by design.
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

__device__ __forceinline__ float ex2_approx(float x) {   // what __expf(x) evaluates after its multiply by log2(e)
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

constexpr int TA_PITCH = 72;   // halves per staged row (64 + 8 pad: conflict-free ldmatrix)
// Persistent: each warp walks (clip, position, head) groups with stride gridDim*4 and keeps the NEXT group's 12 x 16-byte loads in
// flight in registers while it computes the current one. The one-group-per-warp version was latency-bound (ncu: long-scoreboard
// stalls, 47 % occupancy, 23 040 short-lived blocks): 3.0 TB/s.
__global__ void __launch_bounds__(128, 6)
attn_temporal_mma_kernel(const act_t* __restrict__ qkv, int clips, int T, int tokens, int heads, act_t* __restrict__ out) {
    __shared__ __align__(16) act_t sm[4][3][16][TA_PITCH];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t ngroups = (int64_t)clips * tokens * heads, nwarps = (int64_t)gridDim.x * 4;
    const int C = heads * 64;
    const int64_t frame_stride = (int64_t)tokens * 3 * C;
    act_t(*sq)[TA_PITCH] = sm[warp][0];
    act_t(*sk)[TA_PITCH] = sm[warp][1];
    act_t(*sv)[TA_PITCH] = sm[warp][2];
    uint4 pre[12];                                   // 3 matrices x 16 rows x 8 chunks of 16 B, 12 per lane
    auto issue = [&](int64_t g) {
        const int h = (int)(g % heads);
        const int64_t cs = g / heads;
        const act_t* base = qkv + ((cs / tokens) * T * tokens + (cs % tokens)) * 3 * C + h * 64;
#pragma unroll
        for (int i = 0; i < 12; i++) {
            const int idx = i * 32 + lane;
            const int m = idx >> 7, row = (idx >> 3) & 15, ch = idx & 7;
            pre[i] = make_uint4(0, 0, 0, 0);
            if (row < T) pre[i] = *reinterpret_cast<const uint4*>(base + (int64_t)row * frame_stride + m * C + ch * 8);
        }
    };
    int64_t gid = (int64_t)blockIdx.x * 4 + warp;
    if (gid < ngroups) issue(gid);
    for (; gid < ngroups; gid += nwarps) {
    const int h = (int)(gid % heads);
    const int64_t cs = gid / heads;
    const int s = (int)(cs % tokens);
    const int b = (int)(cs / tokens);
    __syncwarp();                                    // the previous group's output staging has been read
#pragma unroll
    for (int i = 0; i < 12; i++) {
        const int idx = i * 32 + lane;
        *reinterpret_cast<uint4*>(&sm[warp][idx >> 7][(idx >> 3) & 15][(idx & 7) * 8]) = pre[i];
    }
    if (gid + nwarps < ngroups) issue(gid + nwarps);  // in flight during the math below
    __syncwarp();
    // ---- S = Q K^T (16 x 16), 4 k-steps over d
    float sc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
    for (int kb = 0; kb < 64; kb += 16) {
        uint32_t a[4], bk[4];
        ldsm_x4(a, &sq[lane & 15][kb + (lane >> 4) * 8]);
        ldsm_x4(bk, &sk[(lane & 7) + ((lane >> 4) << 3)][kb + ((lane >> 3) & 1) * 8]);
        mma16816(sc[0], a, bk[0], bk[1]);
        mma16816(sc[1], a, bk[2], bk[3]);
    }
    // ---- softmax over keys (columns) in the exp2 domain; thread holds rows g, g+8 and columns {2t, 2t+1} + 8*ntile
    const int t2 = (lane & 3) * 2;
    constexpr float SCALE_LOG2 = 0.125f * 1.4426950408889634f;
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 2; nt++) {
#pragma unroll
        for (int e = 0; e < 2; e++) {
            const bool ok = (nt * 8 + t2 + e) < T;
            sc[nt][e] = ok ? sc[nt][e] * SCALE_LOG2 : -INFINITY;
            sc[nt][2 + e] = ok ? sc[nt][2 + e] * SCALE_LOG2 : -INFINITY;
            mx0 = fmaxf(mx0, sc[nt][e]);
            mx1 = fmaxf(mx1, sc[nt][2 + e]);
        }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    // P = 2^15 exp2(s - m), largest 32768: packed to fp16 for P.V, weights down to 2^-40 of the row maximum stay out of the
    // flush-to-zero range (2^-25 without the offset); l carries the same power of two
    mx0 -= 15.f; mx1 -= 15.f;
    float l0 = 0.f, l1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 2; nt++) {
#pragma unroll
        for (int e = 0; e < 2; e++) {
            sc[nt][e] = ex2_approx(sc[nt][e] - mx0); l0 += sc[nt][e];
            sc[nt][2 + e] = ex2_approx(sc[nt][2 + e] - mx1); l1 += sc[nt][2 + e];
        }
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
    uint32_t pa[4] = {pack2(sc[0][0], sc[0][1]), pack2(sc[0][2], sc[0][3]), pack2(sc[1][0], sc[1][1]), pack2(sc[1][2], sc[1][3])};
    // ---- O = P V (16 x 64), one k-step over the 16 keys, 8 n-tiles over d; result staged in the Q tile
    __syncwarp();
#pragma unroll
    for (int d0 = 0; d0 < 64; d0 += 16) {
        uint32_t bv[4];
        ldsm_x4_t(bv, &sv[(lane & 7) + ((lane >> 3) & 1) * 8][d0 + (lane >> 4) * 8]);
        float o0[4] = {0.f, 0.f, 0.f, 0.f}, o1[4] = {0.f, 0.f, 0.f, 0.f};
        mma16816(o0, pa, bv[0], bv[1]);
        mma16816(o1, pa, bv[2], bv[3]);
        const int g = lane >> 2;
        *reinterpret_cast<uint32_t*>(&sq[g][d0 + t2]) = pack2(o0[0] * inv0, o0[1] * inv0);
        *reinterpret_cast<uint32_t*>(&sq[g + 8][d0 + t2]) = pack2(o0[2] * inv1, o0[3] * inv1);
        *reinterpret_cast<uint32_t*>(&sq[g][d0 + 8 + t2]) = pack2(o1[0] * inv0, o1[1] * inv0);
        *reinterpret_cast<uint32_t*>(&sq[g + 8][d0 + 8 + t2]) = pack2(o1[2] * inv1, o1[3] * inv1);
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int idx = i * 32 + lane;
        const int row = idx >> 3, ch = idx & 7;
        if (row < T)
            *reinterpret_cast<uint4*>(out + (((int64_t)b * T + row) * tokens + s) * C + h * 64 + ch * 8) =
                *reinterpret_cast<const uint4*>(&sq[row][ch * 8]);
    }
    }
}

extern "C" int gcd_attention_temporal(const void* qkv, int clips, int T, int tokens, int heads, void* out, void* stream) {
    GCD_REQUIRE(T >= 1 && T <= 32, "attention_temporal: T=%d unsupported (1..32)", T);
    if (T <= 16) {
        const int64_t ngroups = (int64_t)clips * tokens * heads;
        int64_t nb = (ngroups + 3) / 4;
        static int num_sms = 0;
        if (!num_sms) {
            int dev = 0;
            GCD_CUDA_CHECK(cudaGetDevice(&dev));
            GCD_CUDA_CHECK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
        }
        if (nb > (int64_t)num_sms * 6) nb = (int64_t)num_sms * 6;       // persistent: 6 resident blocks per SM
        attn_temporal_mma_kernel<<<(unsigned)nb, 128, 0, (cudaStream_t)stream>>>((const act_t*)qkv, clips, T, tokens, heads,
                                                                               (act_t*)out);
        GCD_CUDA_CHECK(cudaGetLastError());
        g_launches++;
        return 0;
    }
    const int GS = 32;
    const int64_t nthreads = (int64_t)clips * tokens * heads * GS;
    const int64_t blocks = (nthreads + 127) / 128;
    GCD_REQUIRE(blocks < (1ll << 31), "attention_temporal: problem too large");
    if (GS == 16)
        attn_temporal_kernel<16><<<(unsigned)blocks, 128, 0, (cudaStream_t)stream>>>((const act_t*)qkv, clips, T, tokens,
                                                                                     heads, (act_t*)out);
    else
        attn_temporal_kernel<32><<<(unsigned)blocks, 128, 0, (cudaStream_t)stream>>>((const act_t*)qkv, clips, T, tokens,
                                                                                     heads, (act_t*)out);
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches++;
    return 0;
}
