// gcd_b200 — FlashAttention-style spatial self-attention for sm_90a, head_dim 64, wgmma + TMA.
// Reference math: gcd-model/sgm/modules/attention.py:283-344 (CrossAttention.forward, context=None):
//   out = softmax(q k^T / sqrt(64)) v, heads outer in the channel dim ("b n (h d) -> b h n d").
//
// One CTA per (128-query tile, head, frame), three warpgroups:
//   warpgroup 0    : TMA producer (one thread) — the CTA's Q tile once, then K_j / V_j (64 keys each) through a 4-stage
//                    mbarrier ring, all 128B-swizzled.
//   warpgroups 1, 2: 64 query rows each. Per key block: S = Q K_j^T (wgmma m64n64k16, both operands in shared memory,
//                    fp32 S in registers); online softmax in the exp2 domain on the accumulator fragment (each row lives in
//                    the 4 lanes of a quad); P is re-packed in registers as the 16-bit A operand of O += P V_j (wgmma with A
//                    from registers, V as an MN-major B operand). While one warpgroup runs its softmax, the other's MMAs
//                    keep the tensor cores busy.
#include "common.cuh"
#include "../../include/gcd_b200.h"
#include <atomic>
extern std::atomic<int64_t> g_launches;
using namespace ptx;

namespace fa {
constexpr int BQ = 128, BK = 64, D = 64;
constexpr int KV_STAGES = 4;
constexpr int TILE_BYTES = BK * D * 2;       // 8 KB: one 64-row x 64-channel box
constexpr int SMEM = 2 * TILE_BYTES + KV_STAGES * 2 * TILE_BYTES + 256 + 1024;

struct Params {
    int tokens, heads, nblk;
    act_t* out;
};

__device__ __forceinline__ float ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__global__ void __launch_bounds__(384, 1)
attn_kernel(const __grid_constant__ CUtensorMap mapQKV, const Params p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem;                                 // [2 warpgroups][8 KB]
    uint8_t* sK = sQ + 2 * TILE_BYTES;                  // [stage][8 KB]
    uint8_t* sV = sK + KV_STAGES * TILE_BYTES;          // [stage][8 KB]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + KV_STAGES * TILE_BYTES);
    uint64_t* q_full = bars;
    uint64_t* kv_full = bars + 1;                       // KV_STAGES
    uint64_t* kv_empty = kv_full + KV_STAGES;           // KV_STAGES

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * BQ, head = blockIdx.y, frame = blockIdx.z;
    const int C = p.heads * D;
    const int nblk = p.nblk;

    if (threadIdx.x == 0) {
        prefetch_tmap(&mapQKV);
        mbar_init(q_full, 1);
        for (int i = 0; i < KV_STAGES; i++) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 8); }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {
            // ------------------------------------------------ TMA producer (rows past `tokens` are zero-filled)
            mbar_expect_tx(q_full, 2 * TILE_BYTES);
            tma_load_3d(&mapQKV, sQ, q_full, head * D, q0, frame);
            tma_load_3d(&mapQKV, sQ + TILE_BYTES, q_full, head * D, q0 + 64, frame);
            for (int j = 0; j < nblk; j++) {
                const int s = j % KV_STAGES;
                mbar_wait(&kv_empty[s], ((j / KV_STAGES) & 1) ^ 1);
                mbar_expect_tx(&kv_full[s], 2 * TILE_BYTES);
                tma_load_3d(&mapQKV, sK + s * TILE_BYTES, &kv_full[s], C + head * D, j * BK, frame);
                tma_load_3d(&mapQKV, sV + s * TILE_BYTES, &kv_full[s], 2 * C + head * D, j * BK, frame);
            }
        }
        return;
    }
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // ---------------------------------------------------- consumers: 64 query rows per warpgroup
    const int cw = (warp >> 2) - 1;
    const int r0 = cw * 64 + (warp & 3) * 16 + (lane >> 2);    // tile row of this thread's first accumulator row (+8: second)
    const int cb = 2 * (lane & 3);
    constexpr float SCALE_LOG2 = 0.125f * 1.4426950408889634f;
    // P is packed to 16 bits as 2^15 exp(s - m), not exp(s - m): fp16 would flush weights below 2^-25 of the row maximum to 0 (and
    // keep those below 2^-14 as subnormals), losing the mass of many keys 17+ nats below a dominant one. With the offset the
    // largest weight is 32768 < 65504 and the flush threshold drops to 2^-40; l carries the same power of two, so O / l is
    // unchanged. The running maximum m_run is kept shifted by -P_LOG2 (the shift rides on the block maximum's multiply), so the
    // offset costs no instruction; alpha, a difference of two shifted maxima, is the same.
    constexpr float P_LOG2 = 15.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; i++) o[i] = 0.f;
    const uint64_t qd = make_desc_sw128(smem_u32(sQ + cw * TILE_BYTES), 16, 1024);
    mbar_wait(q_full, 0);

    for (int j = 0; j < nblk; j++) {
        const int s = j % KV_STAGES;
        mbar_wait(&kv_full[s], (j / KV_STAGES) & 1);
        // S = Q K_j^T: K tile [64 keys][64 d] is the K-major B operand
        float sv[32];
        const uint64_t kd = make_desc_sw128(smem_u32(sK + s * TILE_BYTES), 16, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; k++) wgmma_m64n64_ss(sv, qd + 2 * k, kd + 2 * k, k != 0);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(sv);

        const int kv_left = p.tokens - j * BK;           // valid keys in this block
        if (kv_left < BK) {
#pragma unroll
            for (int i = 0; i < 8; i++) {
                if (8 * i + cb >= kv_left) { sv[4 * i] = -INFINITY; sv[4 * i + 2] = -INFINITY; }
                if (8 * i + cb + 1 >= kv_left) { sv[4 * i + 1] = -INFINITY; sv[4 * i + 3] = -INFINITY; }
            }
        }
        uint32_t pa[4][4];                               // P as the A operand of the four K=16 steps of P V_j
#pragma unroll
        for (int h = 0; h < 2; h++) {
            float mx = -INFINITY;
#pragma unroll
            for (int i = 0; i < 8; i++) mx = fmaxf(mx, fmaxf(sv[4 * i + 2 * h], sv[4 * i + 2 * h + 1]));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float m_new = fmaxf(m_run[h], fmaf(mx, SCALE_LOG2, -P_LOG2));   // row maximum (log2 units) - P_LOG2
            const float alpha = ex2(m_run[h] - m_new);   // 0 on the first block (m_run = -inf)
            m_run[h] = m_new;
            float ls = 0.f;
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const float e0 = ex2(fmaf(sv[4 * i + 2 * h], SCALE_LOG2, -m_new));   // 2^15 exp(s - m)
                const float e1 = ex2(fmaf(sv[4 * i + 2 * h + 1], SCALE_LOG2, -m_new));
                ls += e0 + e1;
                // accumulator columns 8i..8i+7 = A columns 8(i&1).. of K step i>>1; register 2(i&1) + h
                pa[i >> 1][2 * (i & 1) + h] = pack2(e0, e1);
                o[4 * i + 2 * h] *= alpha;
                o[4 * i + 2 * h + 1] *= alpha;
            }
            l_run[h] = l_run[h] * alpha + ls;
        }
        // O += P V_j: V tile [64 keys][64 d] is an MN-major B operand; a K step of 16 keys = 2048 bytes
        const uint64_t vd = make_desc_sw128(smem_u32(sV + s * TILE_BYTES), 1024, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; k++) wgmma_m64n64_rs_tb(o, pa[k], vd + (uint64_t)(k * 128));
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(o);
        __syncwarp();
        if (lane == 0) mbar_arrive(&kv_empty[s]);
    }
    // ---- epilogue: O / l (row sums completed over the quad)
#pragma unroll
    for (int h = 0; h < 2; h++) {
        float l = l_run[h];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const float inv = 1.0f / l;
        const int row = q0 + r0 + 8 * h;
        if (row >= p.tokens) continue;
        act_t* dst = p.out + ((int64_t)frame * p.tokens + row) * C + head * D + cb;
#pragma unroll
        for (int i = 0; i < 8; i++)
            *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack2(o[4 * i + 2 * h] * inv, o[4 * i + 2 * h + 1] * inv);
    }
}
}  // namespace fa

extern "C" int gcd_attention_spatial(const void* qkv, int frames, int tokens, int heads, void* out, void* stream) {
    GCD_REQUIRE(qkv && out && frames > 0 && tokens > 0 && heads > 0, "attention_spatial: bad arguments");
    GCD_REQUIRE(frames <= 65535 && heads <= 65535, "attention_spatial: grid too large");
    static bool configured = false;
    if (!configured) {
        GCD_CUDA_CHECK(cudaFuncSetAttribute(fa::attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, fa::SMEM));
        configured = true;
    }
    const int C = heads * 64;
    CUtensorMap mQKV;
    uint64_t dims[3] = {(uint64_t)3 * C, (uint64_t)tokens, (uint64_t)frames};
    uint64_t str[2] = {(uint64_t)3 * C * 2, (uint64_t)tokens * 3 * C * 2};
    uint32_t box[3] = {64, 64, 1};
    int rc = gcd_make_tmap(&mQKV, qkv, 3, dims, str, box, nullptr, 128, 0);
    if (rc) return rc;
    fa::Params p;
    p.tokens = tokens; p.heads = heads; p.nblk = (tokens + fa::BK - 1) / fa::BK; p.out = (act_t*)out;
    dim3 grid((tokens + fa::BQ - 1) / fa::BQ, heads, frames);
    fa::attn_kernel<<<grid, 384, fa::SMEM, (cudaStream_t)stream>>>(mQKV, p);
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches++;
    return 0;
}
