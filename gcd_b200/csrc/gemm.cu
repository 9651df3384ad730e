// gcd_b200 — wgmma implicit-GEMM kernel for sm_90a (Linear / Conv2d 3x3 & 1x1 / Conv3d (3,1,1) / batched matmul).
//
// acc[r, n] = sum_{tap, c} A[(x,y,z)(r) * in_mul + tap_off(tap), c] * W[n, tap*C + c], fp16/bf16 operands, fp32 accumulate,
// with the whole epilogue (bias, per-row vector, SiLU, scale, GEGLU, residual blends, GroupNorm statistics) fused.
// Replaces cuDNN/cuBLAS calls behind nn.Conv2d / nn.Conv3d / nn.Linear in
//   gcd-model/sgm/modules/diffusionmodules/openaimodel.py:213-357 (ResBlock), :110-210 (Up/Downsample),
//   gcd-model/sgm/modules/attention.py:87-113,255-344 (FeedForward/GEGLU, CrossAttention projections),
//   gcd-model/sgm/modules/diffusionmodules/model.py:94-201 (VAE ResnetBlock/AttnBlock).
#include "common.cuh"
#include "../../include/gcd_b200.h"
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <atomic>
#include <mutex>
#include <unordered_map>

using namespace ptx;

// ------------------------------------------------------------------------------------------------ host globals
static thread_local char g_err[1024] = "";
std::atomic<int64_t> g_launches{0};
void gcd_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
extern "C" const char* gcd_last_error(void) { return g_err; }
extern "C" int gcd_version(void) { return 101; }
extern "C" int gcd_act_dtype(void) { return (int)GCD_UMMA_FMT; }
extern "C" int64_t gcd_launch_count(void) { return g_launches.load(); }

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (PFN_encodeTiled)p;
    }
    return fn;
}
int gcd_make_tmap(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box, const uint32_t* elem_strides, int swizzle_bytes, int f32) {
    PFN_encodeTiled enc = get_encode();
    GCD_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled driver entry point unavailable (no CUDA driver?)");
    cuuint64_t d[5], s[4];
    cuuint32_t b[5], e[5];
    for (int i = 0; i < rank; i++) {
        d[i] = dims[i];
        b[i] = box[i];
        e[i] = elem_strides ? elem_strides[i] : 1;
    }
    for (int i = 0; i + 1 < rank; i++) s[i] = strides_bytes[i];
#ifdef GCD_ACT_BF16
    CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
#else
    CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
#endif
    if (f32) dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                          : swizzle_bytes == 64  ? CU_TENSOR_MAP_SWIZZLE_64B
                          : swizzle_bytes == 32  ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE;
    CUresult r = enc(out, dt, (cuuint32_t)rank, const_cast<void*>(base), d, s, b, e, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    GCD_REQUIRE(r == CUDA_SUCCESS,
                "cuTensorMapEncodeTiled failed (%d): rank %d dims %llu %llu %llu %llu box %u %u %u %u stride0 %llu f32 %d", (int)r,
                rank, (unsigned long long)d[0], (unsigned long long)(rank > 1 ? d[1] : 0),
                (unsigned long long)(rank > 2 ? d[2] : 0), (unsigned long long)(rank > 3 ? d[3] : 0), b[0],
                rank > 1 ? b[1] : 0, rank > 2 ? b[2] : 0, rank > 3 ? b[3] : 0, (unsigned long long)s[0], f32);
    return 0;
}

// ------------------------------------------------------------------------------------------------ kernel
struct TcParams {
    int ntx, nty, ntz;          // M-tiles along x, y, z
    int lTW, lTH;               // log2 tile extents (TW*TH*TN == 128, or 64 under the ping-pong schedule)
    int Xo, Yo, Zo;             // output extents
    int in_mul;
    int ntaps, kchunks;
    int8_t tdx[9], tdy[9], tdz[9];
    int N, n_tiles;
    int w_batched;
    int stages;                 // smem ring depth
    // epilogue
    const float* bias;
    const float* rowvec;
    int rpv, ldv;
    const void* res1;
    const void* res2;
    int ld1, ld2, r1f32, r2f32;
    float a0, a1, a2;
    void* out;
    int ldo, of32, geglu, act;
    double* gn_stats;           // fused GroupNorm statistics of the output (nullptr: off)
    int gn_cpg, gn_groups;
    long long gn_rpi;
};

constexpr int TC_SMEM_MAX = 232448;            // 227 KB opt-in maximum per CTA
constexpr int TC_THREADS = 384;                // producer warpgroup + two consumer warpgroups
constexpr int TC_BAR_BYTES = 256;              // full[8], empty[8], turn[2] mbarriers

// residuals: plain loads (the output may alias a residual: each element is read, then written, by the same thread).
// `p` points at the first of a column pair; the second is read only when it exists (c1ok).
__device__ __forceinline__ float2 ld_res_pair(const char* p, bool f32, bool c1ok) {
    if (f32) {
        if (c1ok) return *reinterpret_cast<const float2*>(p);
        return make_float2(*reinterpret_cast<const float*>(p), 0.f);
    }
    if (c1ok) return unpack2(*reinterpret_cast<const uint32_t*>(p));
    return make_float2(act2f(*reinterpret_cast<const act_t*>(p)), 0.f);
}

// One persistent, warp-specialised CTA per SM; an M-tile is a TW x TH x TN box of output positions.
//   warpgroup 0 : TMA producer (one thread) — per (tap, 64-channel chunk): one 4-D box of the channels-last activation
//                 tensor (out-of-range coordinates zero-filled by TMA = conv zero padding) + one 3-D box of BN weight rows,
//                 both landing 128B-swizzled in shared memory, signalled on an mbarrier ring. It fills the ring in the
//                 CTA's tile order and runs ahead as far as the ring allows.
//   warpgroups 1, 2 : consumers — wgmma m64nBNk16 (fp32 accumulators in registers, one batch in flight while the previous
//                 stage is released), then the fused epilogue straight from the accumulator registers: bias (+ per-row
//                 vector) / SiLU / scale / GEGLU / two residual blends, 16-bit or fp32 stores, and the GroupNorm statistics
//                 of the stored values. Two schedules:
//     PP = false (cooperative): both work on one 128-row tile, rows [64*cw, +64) each, and run its epilogue together.
//                 Fewest operand bytes per FLOP from L2; the tensor cores idle during the epilogue.
//     PP = true (ping-pong): each owns whole 64 x BN tiles (the CTA's tiles with even / odd local index) and they take
//                 turns on the tensor cores: a warpgroup starts the MMAs of its next tile when the other has issued the
//                 last MMA of its current one, so one runs its epilogue while the other keeps the tensor pipe busy. A
//                 warpgroup finds its stages from the global k-step number (local tile index x k-steps per tile + k-step),
//                 stepping over the stages of the other's tiles. The turn order is also what makes the parity waits on
//                 `full` unambiguous: when a warpgroup starts a tile, every earlier k-step of the CTA has been filled and
//                 waited for, so a stage's barrier cannot still be one ring revolution behind the phase it waits on.
//                 1.67x the operand bytes per FLOP; pays where the epilogue waits on memory (gcd_tc_run chooses).
// ACT: the activation compiled into the epilogue. 0: none or SiLU, chosen at run time by `act` (0 / 1); 2: exact erf GELU;
// 3: ReLU (LPIPS's VGG16). GELU and ReLU are instantiations of their own: the erff expansion inside the unrolled act 0 / 1
// epilogue made the UNet's tc_gemm 14 % slower (same registers; one H100 80GB HBM3 at 400 W). The ACT = 0 instantiations
// compile to the same SASS as without GELU and ReLU.
template <int BN, int ACT, bool PP>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const TcParams p) {
    constexpr int TILE_M = PP ? 64 : 128;
    constexpr int TC_A_BYTES = TILE_M * 128;       // one TILE_M-row x 64-channel activation box, 128B-swizzled
    constexpr int B_BYTES = BN * 128;
    constexpr int STAGE_BYTES = TC_A_BYTES + B_BYTES;
    constexpr int NACC = BN / 2;
    extern __shared__ __align__(1024) uint8_t smem[];     // SWIZZLE_128B tiles need 1024-byte alignment
    if ((smem_u32(smem) & 1023u) != 0) __trap();
    const int STAGES = p.stages;
    float* sStatAll = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);  // [8 consumer warps][BN][sum, sum of squares]; PP: one [4][BN][2] half per warpgroup
    uint64_t* bars = reinterpret_cast<uint64_t*>(sStatAll + (p.gn_stats ? 8 * BN * 2 : 0));
    uint64_t* full = bars;                 // [STAGES]
    uint64_t* empty = bars + 8;            // [STAGES]  (STAGES <= 8)
    uint64_t* turn = bars + 16;            // [2] (PP): turn[w] completes a phase each time warpgroup w may start a main loop

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        prefetch_tmap(&mapA);
        prefetch_tmap(&mapB);
        for (int i = 0; i < STAGES; i++) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], PP ? 4 : 8);   // one arrival per warp that consumed the stage
        }
        mbar_init(&turn[0], 4);
        mbar_init(&turn[1], 4);
        fence_barrier_init();
    }
    __syncthreads();

    const int m_tiles = p.ntx * p.nty * p.ntz;
    const int total = m_tiles * p.n_tiles;
    const int kiters = p.ntaps * p.kchunks;
    const int TW = 1 << p.lTW, TH = 1 << p.lTH;
    const int TN = TILE_M >> (p.lTW + p.lTH);

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {
            // ===================== TMA producer =====================
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
                const int nt = tile % p.n_tiles;
                const int mt = tile / p.n_tiles;
                const int tx = mt % p.ntx;
                const int ty = (mt / p.ntx) % p.nty;
                const int tz = mt / (p.ntx * p.nty);
                const int x0 = tx * TW * p.in_mul, y0 = ty * TH * p.in_mul, z0 = tz * TN;
                const int wy = p.w_batched ? ty : 0;
                for (int q = 0; q < kiters; q++) {
                    const int tap = q / p.kchunks, kc = q - tap * p.kchunks;
                    mbar_wait(&empty[stage], phase ^ 1);
                    mbar_expect_tx(&full[stage], STAGE_BYTES);
                    uint8_t* dA = smem + stage * STAGE_BYTES;
                    tma_load_4d(&mapA, dA, &full[stage], kc * 64, x0 + p.tdx[tap], y0 + p.tdy[tap], z0 + p.tdz[tap]);
                    tma_load_3d(&mapB, dA + TC_A_BYTES, &full[stage], q * 64, nt * BN, wy);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    // ===================== consumers =====================
    const int cw = (warp >> 2) - 1;                 // consumer warpgroup; PP: the CTA's tiles with local index = cw (mod 2)
    const int a_off = PP ? 0 : cw * (64 * 128);     // cooperative: rows [64*cw, +64) of the 128-row activation box
    const int rl = (PP ? 0 : cw * 64) + (warp & 3) * 16 + (lane >> 2);   // tile row of acc[4i], acc[4i+1]; rl + 8: acc[4i+2], acc[4i+3]
    const int cb = 2 * (lane & 3);
    // statistics party: the threads that share one table and one stream of tiles (a warpgroup under PP, else both)
    constexpr int ST_WARPS = PP ? 4 : 8, ST_THREADS = ST_WARPS * 32;
    const int st_t = PP ? (threadIdx.x & 127) : threadIdx.x - 128;
    const int st_w = PP ? (warp & 3) : warp - 4;
    const int st_bar = PP ? 1 + cw : 1;
    float* sStat = sStatAll + (PP ? cw * (4 * BN * 2) : 0);
    // GroupNorm statistics: party thread g < gn_groups owns group g of the party's current image and flushes it
    // (fp64 atomics) when its tile stream moves to another image — tiles of one image are many, the atomics per image few.
    int cur_img = -1;
    double st1 = 0.0, st2 = 0.0;
    auto flush = [&]() {
        if (cur_img >= 0 && st_t < p.gn_groups && (st1 != 0.0 || st2 != 0.0)) {
            double* dst = p.gn_stats + ((int64_t)cur_img * p.gn_groups + st_t) * 2;
            atomicAdd(dst, st1);
            atomicAdd(dst + 1, st2);
        }
        st1 = st2 = 0.0;
    };

    float acc[NACC];
    uint32_t turn_parity = cw ^ 1;                  // warpgroup 0 starts at once (parity of the phase before the first)
    for (int j = PP ? cw : 0;; j += PP ? 2 : 1) {
        const int tile = blockIdx.x + j * gridDim.x;
        if (tile >= total) break;
        const int nt = tile % p.n_tiles;
        const int mt = tile / p.n_tiles;
        const int tx = mt % p.ntx;
        const int ty = (mt / p.ntx) % p.nty;
        const int tz = mt / (p.ntx * p.nty);
        const int n0 = nt * BN;
        const int g0 = j * kiters;                  // global k-step number of the tile's first stage
        int stage = g0 % STAGES;
        uint32_t phase = (g0 / STAGES) & 1;
#pragma unroll
        for (int i = 0; i < NACC; i++) acc[i] = 0.f;
        if constexpr (PP) {
            mbar_wait(&turn[cw], turn_parity);
            turn_parity ^= 1;
        }
        int prev = -1;
        for (int q = 0; q < kiters; q++) {
            mbar_wait(&full[stage], phase);
            const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
            const uint64_t ad = make_desc_sw128(sa + a_off, 16, 1024);
            const uint64_t bd = make_desc_sw128(sa + TC_A_BYTES, 16, 1024);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; k++) {           // 4 x (K=16) inside the 64-wide swizzle atom: +32 B each
                if constexpr (BN == 256) wgmma_m64n256_ss(acc, ad + 2 * k, bd + 2 * k, 1u);
                else if constexpr (BN == 160) wgmma_m64n160_ss(acc, ad + 2 * k, bd + 2 * k, 1u);
                else wgmma_m64n128_ss(acc, ad + 2 * k, bd + 2 * k, 1u);
            }
            wgmma_commit();
            if (PP && q + 1 == kiters && lane == 0) mbar_arrive(&turn[cw ^ 1]);    // last MMA issued: the other warpgroup's turn
            wgmma_wait<1>();                        // the previous stage's batch is done: release its buffers
            if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
            prev = stage;
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        fence_regs(acc);
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);

        // ---- epilogue: output rows of this thread (-1: outside the output)
        int64_t grow[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int r = rl + 8 * h;
            const int x = tx * TW + (r & (TW - 1));
            const int y = ty * TH + ((r >> p.lTW) & (TH - 1));
            const int z = tz * TN + (r >> (p.lTW + p.lTH));
            grow[h] = (x < p.Xo && y < p.Yo && z < p.Zo) ? ((int64_t)z * p.Yo + y) * p.Xo + x : -1;
        }
        if (p.geglu) {
            // value columns 32b + [0,16), gate columns 32b + [16,32) of the accumulator -> output columns 16b + [0,16)
            act_t* out = reinterpret_cast<act_t*>(p.out);
#pragma unroll
            for (int i = 0; i < BN / 8; i++) {
                if ((i & 3) >= 2) continue;
                const int col = n0 + 8 * i + cb;
                const float2 bv = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + col)) : make_float2(0.f, 0.f);
                const float2 bg = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + col + 16)) : make_float2(0.f, 0.f);
                const int oc = (n0 >> 1) + 16 * (i >> 2) + 8 * (i & 3) + cb;
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    if (grow[h] < 0) continue;
                    const float o0 = geglu(acc[4 * i + 2 * h] + bv.x, acc[4 * (i + 2) + 2 * h] + bg.x);
                    const float o1 = geglu(acc[4 * i + 2 * h + 1] + bv.y, acc[4 * (i + 2) + 2 * h + 1] + bg.y);
                    *reinterpret_cast<uint32_t*>(out + grow[h] * p.ldo + oc) = pack2(o0, o1);
                }
            }
            continue;
        }
        const float* bias = p.bias ? p.bias + n0 + cb : nullptr;    // this thread's first column
        // row base pointers (bytes) of this thread's first column, once per tile; column group i adds 8 * i elements
        const int eso = p.of32 ? 4 : 2, es1 = p.r1f32 ? 4 : 2, es2 = p.r2f32 ? 4 : 2;
        char* orow[2];
        const char* r1row[2];
        const char* r2row[2];
        const float* rv[2] = {nullptr, nullptr};
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int64_t g = grow[h] < 0 ? 0 : grow[h];
            orow[h] = reinterpret_cast<char*>(p.out) + (g * p.ldo + n0 + cb) * eso;
            r1row[h] = reinterpret_cast<const char*>(p.res1) + (g * p.ld1 + n0 + cb) * es1;
            r2row[h] = reinterpret_cast<const char*>(p.res2) + (g * p.ld2 + n0 + cb) * es2;
            if (p.rowvec && grow[h] >= 0) rv[h] = p.rowvec + (grow[h] / p.rpv) * (int64_t)p.ldv + n0 + cb;
        }
        const bool stats = p.gn_stats != nullptr;
        const bool has1 = p.res1 != nullptr, has2 = p.res2 != nullptr;
        // residuals of column group i are loaded one group ahead of the arithmetic that uses them
        float2 t1[2], t2[2];
        auto load_res = [&](int i, float2 (&a)[2], float2 (&b)[2]) {
            const int col = n0 + 8 * i + cb;
            if (col >= p.N) return;
            const bool c1ok = col + 1 < p.N;
#pragma unroll
            for (int h = 0; h < 2; h++) {
                if (grow[h] < 0) continue;
                if (has1) a[h] = ld_res_pair(r1row[h] + 8 * i * es1, p.r1f32, c1ok);
                if (has2) b[h] = ld_res_pair(r2row[h] + 8 * i * es2, p.r2f32, c1ok);
            }
        };
        t1[0] = t1[1] = t2[0] = t2[1] = make_float2(0.f, 0.f);
        load_res(0, t1, t2);
#pragma unroll
        for (int i = 0; i < BN / 8; i++) {
            const int col = n0 + 8 * i + cb;
            const bool c0ok = col < p.N, c1ok = col + 1 < p.N;
            float2 u1[2] = {t1[0], t1[1]}, u2[2] = {t2[0], t2[1]};
            if (i + 1 < BN / 8) load_res(i + 1, t1, t2);
            float s1a = 0.f, s2a = 0.f, s1b = 0.f, s2b = 0.f;   // statistics of columns col, col + 1 over this thread's rows
            if (c0ok) {
                float2 b = make_float2(0.f, 0.f);
                if (bias) b = c1ok ? __ldg(reinterpret_cast<const float2*>(bias + 8 * i)) : make_float2(__ldg(bias + 8 * i), 0.f);
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    if (grow[h] < 0) continue;
                    float v0 = acc[4 * i + 2 * h] + b.x, v1 = acc[4 * i + 2 * h + 1] + b.y;
                    if (rv[h]) { v0 += rv[h][8 * i]; if (c1ok) v1 += rv[h][8 * i + 1]; }
                    if constexpr (ACT == 2) { v0 = gelu_erf(v0); v1 = gelu_erf(v1); }
                    else if constexpr (ACT == 3) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                    else if (p.act == 1) { v0 = silu(v0); v1 = silu(v1); }
                    v0 *= p.a0; v1 *= p.a0;
                    if (has1) { v0 += p.a1 * u1[h].x; if (c1ok) v1 += p.a1 * u1[h].y; }
                    if (has2) { v0 += p.a2 * u2[h].x; if (c1ok) v1 += p.a2 * u2[h].y; }
                    char* o = orow[h] + 8 * i * eso;
                    if (p.of32) {
                        if (c1ok) *reinterpret_cast<float2*>(o) = make_float2(v0, v1);
                        else *reinterpret_cast<float*>(o) = v0;
                    } else {
                        const uint32_t w = pack2(v0, v1);
                        if (c1ok) *reinterpret_cast<uint32_t*>(o) = w;
                        else *reinterpret_cast<act_t*>(o) = f2act(v0);
                        const float2 r = unpack2(w);             // statistics of the stored (rounded) values
                        v0 = r.x; v1 = r.y;
                    }
                    s1a += v0; s2a += v0 * v0;
                    if (c1ok) { s1b += v1; s2b += v1 * v1; }
                }
            }
            if (stats) {                            // fold the 8 row-groups of the warp (lanes with equal lane % 4)
#pragma unroll
                for (int off = 4; off < 32; off <<= 1) {
                    s1a += __shfl_xor_sync(0xffffffffu, s1a, off); s2a += __shfl_xor_sync(0xffffffffu, s2a, off);
                    s1b += __shfl_xor_sync(0xffffffffu, s1b, off); s2b += __shfl_xor_sync(0xffffffffu, s2b, off);
                }
                if (lane < 4) {
                    float* d = sStat + (st_w * BN + 8 * i + cb) * 2;
                    d[0] = s1a; d[1] = s2a; d[2] = s1b; d[3] = s2b;
                }
            }
        }
        if (stats) {
            // fixed summation order (warps, then columns of the group): the statistics do not depend on scheduling.
            // The barrier spans the statistics party only: under PP the other warpgroup is in its main loop.
            named_bar_sync(st_bar, ST_THREADS);
            for (int c = st_t; c < BN; c += ST_THREADS) {
                float a = 0.f, b = 0.f;
#pragma unroll
                for (int w = 0; w < ST_WARPS; w++) { a += sStat[(w * BN + c) * 2]; b += sStat[(w * BN + c) * 2 + 1]; }
                sStat[c * 2] = a; sStat[c * 2 + 1] = b;
            }
            named_bar_sync(st_bar, ST_THREADS);
            const int64_t row0 = ((int64_t)(tz * TN) * p.Yo + ty * TH) * p.Xo + tx * TW;
            const int img = (int)(row0 / p.gn_rpi);
            if (img != cur_img) { flush(); cur_img = img; }
            if (st_t < p.gn_groups) {
                const int lo = max(st_t * p.gn_cpg, n0), hi = min(min((st_t + 1) * p.gn_cpg, n0 + BN), p.N);
                for (int c = lo; c < hi; c++) { st1 += (double)sStat[(c - n0) * 2]; st2 += (double)sStat[(c - n0) * 2 + 1]; }
            }
            named_bar_sync(st_bar, ST_THREADS);     // sStat is rewritten by the next tile
        }
    }
    if (p.gn_stats) flush();
}

// ------------------------------------------------------------------------------------------------ host launcher
static int ilog2(int v) {
    int l = 0;
    while ((1 << l) < v) l++;
    return l;
}

static int num_sms_cached() {
    static const int n = [] { int d = 0, v = 0; cudaGetDevice(&d); cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d); return v; }();
    return n;
}

template <int BN, int ACT, bool PP>
static int launch_tc(const CUtensorMap& mA, const CUtensorMap& mB, TcParams& p, cudaStream_t st) {
    static bool configured = false;
    if (!configured) {
        GCD_CUDA_CHECK(cudaFuncSetAttribute(tc_gemm_kernel<BN, ACT, PP>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_MAX));
        configured = true;
    }
    constexpr int STAGE_BYTES = (PP ? 64 : 128) * 128 + BN * 128;
    const int fixed = (p.gn_stats ? 8 * BN * 2 * 4 : 0) + TC_BAR_BYTES;     // statistics tables + barriers
    int stages = (TC_SMEM_MAX - fixed) / STAGE_BYTES;
    if (stages > 8) stages = 8;
    GCD_REQUIRE(stages >= 2, "tc_gemm: not enough shared memory for the pipeline (BN=%d)", BN);
    p.stages = stages;
    const int smem = stages * STAGE_BYTES + fixed;
    const int tiles = p.ntx * p.nty * p.ntz * p.n_tiles;
    const int sms = num_sms_cached();
    GCD_REQUIRE(sms > 0, "tc_gemm: no CUDA device");
    const int grid = tiles < sms ? tiles : sms;
    tc_gemm_kernel<BN, ACT, PP><<<grid, TC_THREADS, smem, st>>>(mA, mB, p);
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches++;
    return 0;
}

// 16-byte alignment of an epilogue tensor and its rows (vector loads / stores of column pairs)
static int check_ep_tensor(const void* ptr, int f32, int ld, const char* what) {
    const int es = f32 ? 4 : 2;
    GCD_REQUIRE(((uintptr_t)ptr & 15) == 0 && ((int64_t)ld * es) % 16 == 0,
                "gcd_tc_run: %s must be 16-byte aligned with a leading dimension multiple of 16 bytes (ld=%d)", what, ld);
    return 0;
}

// ---- tensor-map cache (host)
struct TmapKey { gcd_tc_op op; int bn; };
struct TmapSet { CUtensorMap m[2]; };
struct TmapKeyHash {
    size_t operator()(const TmapKey& k) const {
        const unsigned char* b = reinterpret_cast<const unsigned char*>(&k);
        uint64_t h = 1469598103934665603ull;                                  // FNV-1a over the (zero-initialised) key bytes
        for (size_t i = 0; i < sizeof(TmapKey); i++) { h ^= b[i]; h *= 1099511628211ull; }
        return (size_t)h;
    }
};
struct TmapKeyEq { bool operator()(const TmapKey& a, const TmapKey& b) const { return memcmp(&a, &b, sizeof(TmapKey)) == 0; } };
static std::mutex g_tmap_mu;
static std::unordered_map<TmapKey, TmapSet, TmapKeyHash, TmapKeyEq> g_tmap_cache;
static bool tmap_cache_find(const TmapKey& k, TmapSet* out) {
    std::lock_guard<std::mutex> lk(g_tmap_mu);
    auto it = g_tmap_cache.find(k);
    if (it == g_tmap_cache.end()) return false;
    *out = it->second;
    return true;
}
static void tmap_cache_put(const TmapKey& k, const TmapSet& v) {
    std::lock_guard<std::mutex> lk(g_tmap_mu);
    if (g_tmap_cache.size() >= 8192) g_tmap_cache.clear();                    // bounded: a new shape set simply refills it
    g_tmap_cache.emplace(k, v);
}

// Experiments only (tools/autotune_tc.py): force the tile width of the following gcd_tc_run calls (0 = automatic; `mode` is ignored).
static int g_ovr_bn = 0;
extern "C" void gcd_tc_override(int bn, int mode) { g_ovr_bn = bn; (void)mode; }

extern "C" int gcd_tc_run(const gcd_tc_op* op, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    GCD_REQUIRE(op && op->A && op->W && op->ep.out, "gcd_tc_run: null pointer");
    GCD_REQUIRE(op->ntaps >= 1 && op->ntaps <= 9, "gcd_tc_run: ntaps %d out of range", op->ntaps);
    GCD_REQUIRE(op->C % 8 == 0 && op->C > 0, "gcd_tc_run: C=%d must be a positive multiple of 8", op->C);
    GCD_REQUIRE(op->sx % 8 == 0 && op->sy % 8 == 0 && op->sz % 8 == 0 && op->ldw % 8 == 0,
                "gcd_tc_run: strides must be multiples of 8 elements (16 B)");
    GCD_REQUIRE(((uintptr_t)op->A & 15) == 0 && ((uintptr_t)op->W & 15) == 0, "gcd_tc_run: operands must be 16B aligned");
    GCD_REQUIRE(op->in_mul == 1 || op->in_mul == 2, "gcd_tc_run: in_mul must be 1 or 2");
    const gcd_epilogue& e = op->ep;
    GCD_REQUIRE(!e.geglu || (op->N % 256 == 0 && !e.out_f32 && !e.res1 && !e.res2 && e.a_acc == 1.0f && !e.act),
                "gcd_tc_run: GEGLU needs N %% 256 == 0, 16-bit output, no residual / scale / activation");
    GCD_REQUIRE(e.act >= 0 && e.act <= 3, "gcd_tc_run: act=%d unsupported (0 none, 1 SiLU, 2 GELU, 3 ReLU)", e.act);
    GCD_REQUIRE(!e.rowvec || e.rows_per_vec > 0, "gcd_tc_run: rows_per_vec must be > 0");
    GCD_REQUIRE(!e.bias || ((uintptr_t)e.bias & 15) == 0, "gcd_tc_run: bias must be 16B aligned");
    GCD_REQUIRE(!e.rowvec || (((uintptr_t)e.rowvec & 15) == 0 && e.ld_rowvec % 4 == 0),
                "gcd_tc_run: rowvec must be 16B aligned with ld %% 4 == 0");

    TcParams p;
    memset(&p, 0, sizeof(p));
    // ---- schedule. Ping-pong hides an epilogue that waits on memory (residual reads, fp32 stores) behind the other
    // warpgroup's MMAs, at 1.67x the operand bytes per FLOP from L2. Measured per op of the UNet forward and the VAE decode on
    // one H100 80GB HBM3 at a 700 W limit: ops with a residual or an fp32 output 14-40 % faster under ping-pong, plain 16-bit
    // stores within a few per cent either way; the GEGLU GEMMs already run at 420-600 TFLOP/s cooperatively (DESIGN.md §6).
    const bool pp = !e.geglu && (e.res1 || e.res2 || e.out_f32);
    const int TILE_M = pp ? 64 : 128;
    // ---- tile search
    int TW, TH, TN;
    if (op->gemm_tile) {
        TW = TILE_M; TH = 1; TN = 1;
    } else {
        TW = 1;
        while (TW < TILE_M && op->Xo % (TW * 2) == 0) TW *= 2;
        long best = -1;
        int bestTH = 1;
        for (int th = 1; th * TW <= TILE_M; th *= 2) {
            int tn = TILE_M / (TW * th);
            long cov = (long)((op->Yo + th - 1) / th) * th * (long)((op->Zo + tn - 1) / tn) * tn;
            if (best < 0 || cov <= best) { best = cov; bestTH = th; }
        }
        TH = bestTH;
        TN = TILE_M / (TW * TH);
    }
    p.lTW = ilog2(TW);
    p.lTH = ilog2(TH);
    p.ntx = (op->Xo + TW - 1) / TW;
    p.nty = (op->Yo + TH - 1) / TH;
    p.ntz = (op->Zo + TN - 1) / TN;
    p.Xo = op->Xo; p.Yo = op->Yo; p.Zo = op->Zo;
    p.in_mul = op->in_mul;
    p.ntaps = op->ntaps;
    p.kchunks = (op->C + 63) / 64;
    for (int i = 0; i < op->ntaps; i++) { p.tdx[i] = op->tap_dx[i]; p.tdy[i] = op->tap_dy[i]; p.tdz[i] = op->tap_dz[i]; }
    p.N = op->N;
    p.w_batched = op->w_batch_stride != 0;
    GCD_REQUIRE(!p.w_batched || TH == 1, "gcd_tc_run: batched weights need gemm tiling");

    // Tile width: the widest wgmma (N = 256) reads each activation tile once per 256 output columns; N = 320 / 640 / 1280
    // convs split evenly into 160-column tiles. On small problems (the 9x16 / 18x32 levels: M = 4032 rows = 63 M-tiles) wave
    // quantisation over the SMs decides instead: cost = waves x tile width.
    int BN;
    if (op->N % 256 == 0 || op->N >= 384) BN = 256;
    else if (op->N % 160 == 0) BN = 160;
    else BN = 128;
    const int num_sms_h = num_sms_cached();
    GCD_REQUIRE(num_sms_h > 0, "gcd_tc_run: no CUDA device");
    if (BN == 256 && !e.geglu && op->N % 160 == 0) {
        const long m_tiles = (long)p.ntx * p.nty * p.ntz;
        auto cost = [&](int bn) { return (double)((m_tiles * ((op->N + bn - 1) / bn) + num_sms_h - 1) / num_sms_h) * bn; };
        if (cost(160) < 0.9 * cost(256)) BN = 160;
    }
    if ((g_ovr_bn == 128 || g_ovr_bn == 160 || g_ovr_bn == 256) && !e.geglu) BN = g_ovr_bn;
    p.n_tiles = (op->N + BN - 1) / BN;

    p.bias = e.bias; p.rowvec = e.rowvec; p.rpv = e.rows_per_vec; p.ldv = e.ld_rowvec;
    p.res1 = e.res1; p.res2 = e.res2; p.ld1 = e.ld_res1; p.ld2 = e.ld_res2; p.r1f32 = e.res1_f32; p.r2f32 = e.res2_f32;
    p.a0 = e.a_acc; p.a1 = e.a_res1; p.a2 = e.a_res2;
    p.out = e.out; p.ldo = e.ld_out; p.of32 = e.out_f32; p.geglu = e.geglu; p.act = e.act;
    if (check_ep_tensor(e.out, e.out_f32, e.ld_out, "out")) return -2;
    if (e.res1 && check_ep_tensor(e.res1, e.res1_f32, e.ld_res1, "res1")) return -2;
    if (e.res2 && check_ep_tensor(e.res2, e.res2_f32, e.ld_res2, "res2")) return -2;
    int stats_skipped = 0;
    if (e.gn_stats) {
        GCD_REQUIRE(e.gn_cpg > 0 && e.gn_groups > 0 && e.gn_groups <= 128 && e.gn_rows_per_img > 0 && !e.geglu,
                    "gcd_tc_run: bad gn_stats arguments (at most 128 groups: one thread of a consumer warpgroup per group)");
        const long long rpi = e.gn_rows_per_img, plane = (long long)op->Xo * op->Yo;
        const bool full = (op->Xo % TW == 0) && (op->Yo % TH == 0) && (op->Zo % TN == 0);
        const bool one_img = TN == 1 && ((rpi % plane == 0) || (TH == 1 && rpi % TW == 0 && (op->Xo % rpi == 0 || rpi % op->Xo == 0)));
        if (full && one_img) { p.gn_stats = e.gn_stats; p.gn_cpg = e.gn_cpg; p.gn_groups = e.gn_groups; p.gn_rpi = rpi; }
        else stats_skipped = 1;
    }

    // ---- tensor maps: two cuTensorMapEncodeTiled calls per op, cached per (descriptor, tile width) — every forward
    // of the eager paths (VAE decode, generic sampler path, the capture pass of the CUDA graph) re-issues the same few hundred ops
    // on the same pool buffers. The key is the whole gcd_tc_op (pointers, extents, strides, epilogue tensors) + BN.
    CUtensorMap mA, mB;
    TmapKey tkey;
    memset(&tkey, 0, sizeof(tkey));
    tkey.op = *op; tkey.bn = BN;
    tkey.op.ep.a_acc = tkey.op.ep.a_res1 = tkey.op.ep.a_res2 = 0.f;           // scalars / non-tensor fields do not shape the maps
    tkey.op.ep.bias = nullptr; tkey.op.ep.rowvec = nullptr; tkey.op.ep.gn_stats = nullptr;
    tkey.op.ep.rows_per_vec = tkey.op.ep.ld_rowvec = 0; tkey.op.ep.act = 0; tkey.op.ep.gn_cpg = tkey.op.ep.gn_groups = 0; tkey.op.ep.gn_rows_per_img = 0;
    TmapSet hit;
    if (tmap_cache_find(tkey, &hit)) {
        mA = hit.m[0]; mB = hit.m[1];
    } else {
    {
        uint64_t dims[4] = {(uint64_t)op->C, (uint64_t)op->Xi, (uint64_t)op->Yi, (uint64_t)op->Zi};
        uint64_t str[3] = {(uint64_t)op->sx * 2, (uint64_t)op->sy * 2, (uint64_t)op->sz * 2};
        uint32_t box[4] = {64, (uint32_t)TW, (uint32_t)TH, (uint32_t)TN};
        uint32_t es[4] = {1, 1, 1, 1};
        if (op->in_mul == 2) {   // box spans 2*T-1 source elements traversed with stride 2 -> exactly T samples
            if (TW > 1) { box[1] = 2 * TW - 1; es[1] = 2; }
            if (TH > 1) { box[2] = 2 * TH - 1; es[2] = 2; }
        }
        for (int i = 0; i < 3; i++) if (str[i] == 0) str[i] = 16;
        int rc = gcd_make_tmap(&mA, op->A, 4, dims, str, box, es, 128, 0);
        if (rc) return rc;
    }
    {
        uint64_t nb = p.w_batched ? (uint64_t)op->Yo : 1;
        GCD_REQUIRE(op->C % 64 == 0 || op->ntaps == 1, "gcd_tc_run: multi-tap ops need C %% 64 == 0 (got %d)", op->C);
        uint64_t dims[3] = {(uint64_t)op->ntaps * (uint64_t)op->C, (uint64_t)op->N, nb};
        uint64_t str[2] = {(uint64_t)op->ldw * 2, (uint64_t)(p.w_batched ? op->w_batch_stride : op->ldw * (int64_t)op->N) * 2};
        uint32_t box[3] = {64, (uint32_t)BN, 1};
        int rc = gcd_make_tmap(&mB, op->W, 3, dims, str, box, nullptr, 128, 0);
        if (rc) return rc;
    }
    TmapSet ts;
    ts.m[0] = mA; ts.m[1] = mB;
    tmap_cache_put(tkey, ts);
    }
    int rc;
#define GCD_TC_LAUNCH_ACT(bn, a) (pp ? launch_tc<bn, a, true>(mA, mB, p, st) : launch_tc<bn, a, false>(mA, mB, p, st))
#define GCD_TC_LAUNCH(bn)                                                                                  \
    (e.act == 2 ? GCD_TC_LAUNCH_ACT(bn, 2) : e.act == 3 ? GCD_TC_LAUNCH_ACT(bn, 3) : GCD_TC_LAUNCH_ACT(bn, 0))
    switch (BN) {
        case 256: rc = GCD_TC_LAUNCH(256); break;
        case 160: rc = GCD_TC_LAUNCH(160); break;
        default: rc = GCD_TC_LAUNCH(128); break;
    }
#undef GCD_TC_LAUNCH
#undef GCD_TC_LAUNCH_ACT
    return rc ? rc : stats_skipped;
}
