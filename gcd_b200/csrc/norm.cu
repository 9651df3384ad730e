// gcd_b200 — HBM-bound normalisation kernels on channels-last tensors.
//   GroupNorm32 / Normalize : gcd-model/sgm/modules/diffusionmodules/util.py:259-276, attention.py:125-128,
//                             model.py:52-55 (computed in fp32 like GroupNorm32.forward's x.float()).
//   LayerNorm               : attention.py:456-572 (norm1-3), video_attention.py:15-143 (norm_in, norm1-3).
// Roofline: pure streaming; stats pass reads the tensor once, apply pass reads once + writes act once.
#include "common.cuh"
#include "../../include/gcd_b200.h"
#include <atomic>
extern std::atomic<int64_t> g_launches;

// ---------------------------------------------------------------------------------------------- GroupNorm stats
// grid: (row_chunks, n_img). block: (C/4, RY). Each thread owns 4 consecutive channels = 2 channel pairs
// (a pair never straddles a group because C/groups is even).
//
// Accuracy: the consumer derives var = sum(x^2)/n - mean^2, whose two terms are both about mean^2, so the sums are kept in
// fp64 from each element on (fp32 partials lost the difference for groups whose mean is large against their spread:
// |mean|/std = 1e3 cost ~1e-2 of rstd). The square of an fp32 value is exact in fp64.
// Determinism (no floating-point smem atomics: run-to-run bit differences in the statistics flipped 16-bit roundings
// downstream): per-thread partials -> smem [RY][C/2 pairs] -> one thread per group folds its pairs in a fixed order -> one
// fp64 atomic per (block, group) and moment. Before the atomic, each block rounds its two sums to multiples of 2^-26 rms and
// 2^-26 rms^2 (rms of the block's group values, rounded down to a power of two), so blocks of similar rms add values on a
// common grid, exactly and in any order, while the rounding stays far below the accuracy the consumer needs.
__device__ __forceinline__ void gn_block_stats(const double* sm, int npairs, int cpg, int groups, int64_t nrows,
                                               double* __restrict__ st) {
    const int tid = threadIdx.y * blockDim.x + threadIdx.x;
    if (tid >= groups) return;
    const int ppg = cpg >> 1;                          // channel pairs per group
    double s = 0.0, q = 0.0;
    for (int y = 0; y < (int)blockDim.y; y++) {
        const double* row = sm + ((size_t)y * npairs + (size_t)tid * ppg) * 2;
        for (int pp = 0; pp < ppg; pp++) { s += row[2 * pp]; q += row[2 * pp + 1]; }
    }
    if (q > 0.0 && q <= 1e300) {
        const int e = ilogb(q / ((double)nrows * cpg)) >> 1;     // ~log2(rms)
        s = ldexp(rint(ldexp(s, 26 - e)), e - 26);
        q = ldexp(rint(ldexp(q, 26 - 2 * e)), 2 * e - 26);
    }
    atomicAdd(&st[tid * 2 + 0], s);
    atomicAdd(&st[tid * 2 + 1], q);
}

template <bool IN_F32>
__global__ void gn_stats_kernel(const void* __restrict__ in, int64_t rows, int C, int cpg, int rows_per_block,
                                double* __restrict__ stats, int groups) {
    extern __shared__ double sm[];                     // [blockDim.y][C/2][2]
    const int img = blockIdx.y;
    const int c = threadIdx.x * 4;
    const int64_t r0 = (int64_t)blockIdx.x * rows_per_block;
    const int64_t r1 = min(rows, r0 + rows_per_block);
    double sa = 0.0, qa = 0.0, sb = 0.0, qb = 0.0;
#pragma unroll 4
    for (int64_t r = r0 + threadIdx.y; r < r1; r += blockDim.y) {
        const int64_t off = ((int64_t)img * rows + r) * C + c;
        float x0, x1, x2, x3;
        if (IN_F32) {
            float4 v = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(in) + off);
            x0 = v.x; x1 = v.y; x2 = v.z; x3 = v.w;
        } else {
            uint2 v = *reinterpret_cast<const uint2*>(reinterpret_cast<const act_t*>(in) + off);
            float2 a = unpack2(v.x), b = unpack2(v.y);
            x0 = a.x; x1 = a.y; x2 = b.x; x3 = b.y;
        }
        const double d0 = x0, d1 = x1, d2 = x2, d3 = x3;
        sa += d0 + d1; qa += d0 * d0 + d1 * d1;
        sb += d2 + d3; qb += d2 * d2 + d3 * d3;
    }
    const int npairs = C >> 1;
    double* mine = sm + ((size_t)threadIdx.y * npairs + 2 * threadIdx.x) * 2;
    mine[0] = sa; mine[1] = qa; mine[2] = sb; mine[3] = qb;
    __syncthreads();
    gn_block_stats(sm, npairs, cpg, groups, r1 - r0, stats + (int64_t)img * groups * 2);
}

// Channel concat of two fp32 tensors fused with the GroupNorm statistics of the result (the UNet's skip concatenations,
// openaimodel.py `th.cat([h, hs.pop()], dim=1)` followed by the ResBlock's first GroupNorm): same geometry and the same
// deterministic fp64 reduction as gn_stats_kernel; saves the statistics pass over the concatenated tensor.
// OUT_ACT: the concatenated tensor is written in the 16-bit activation type only — the consumer ResBlock always has
// cin != cout there (its 1x1 skip conv and its first GroupNorm read 16-bit operands; nothing reads the fp32 concat), which removes
// the fp32 write of the concat, the fp32 read of the GroupNorm and the separate cast pass: 20 -> 10 bytes per element.
// The statistics are those of the fp32 inputs, like the tensor-core epilogues' (sums of the values before the 16-bit rounding).
template <bool OUT_ACT>
__global__ void concat_stats_kernel(const float* __restrict__ a, int Ca, const float* __restrict__ b, int Cb, int64_t rows,
                                    int cpg, int rows_per_block, void* __restrict__ out_, double* __restrict__ stats,
                                    int groups) {
    extern __shared__ double sm[];                     // [blockDim.y][C/2][2]
    const int img = blockIdx.y;
    const int C = Ca + Cb;
    const int c = threadIdx.x * 4;
    const bool from_a = c < Ca;                        // Ca is a multiple of 4: a thread's 4 channels come from one source
    const float* src = from_a ? a + c : b + (c - Ca);
    const int ld = from_a ? Ca : Cb;
    const int64_t r0 = (int64_t)blockIdx.x * rows_per_block;
    const int64_t r1 = min(rows, r0 + rows_per_block);
    double sa = 0.0, qa = 0.0, sb = 0.0, qb = 0.0;
#pragma unroll 4
    for (int64_t r = r0 + threadIdx.y; r < r1; r += blockDim.y) {
        const int64_t row = (int64_t)img * rows + r;
        const float4 v = *reinterpret_cast<const float4*>(src + row * ld);
        if (OUT_ACT) *reinterpret_cast<uint2*>(reinterpret_cast<act_t*>(out_) + row * C + c) = make_uint2(pack2(v.x, v.y), pack2(v.z, v.w));
        else *reinterpret_cast<float4*>(reinterpret_cast<float*>(out_) + row * C + c) = v;
        const double d0 = v.x, d1 = v.y, d2 = v.z, d3 = v.w;
        sa += d0 + d1; qa += d0 * d0 + d1 * d1;
        sb += d2 + d3; qb += d2 * d2 + d3 * d3;
    }
    const int npairs = C >> 1;
    double* mine = sm + ((size_t)threadIdx.y * npairs + 2 * threadIdx.x) * 2;
    mine[0] = sa; mine[1] = qa; mine[2] = sb; mine[3] = qb;
    __syncthreads();
    gn_block_stats(sm, npairs, cpg, groups, r1 - r0, stats + (int64_t)img * groups * 2);
}

template <bool IN_F32>
__global__ void gn_apply_kernel(const void* __restrict__ in, int64_t rows, int C, int cpg, int rows_per_block,
                                const double* __restrict__ stats, int groups, const float* __restrict__ gamma,
                                const float* __restrict__ beta, float eps, int do_silu, act_t* __restrict__ out) {
    const int img = blockIdx.y;
    const int c = threadIdx.x * 4;
    const int ga = c / cpg, gb = (c + 2) / cpg;
    const double cnt = (double)rows * (double)cpg;
    float ma, ra, mb, rb;
    {
        double s = stats[((int64_t)img * groups + ga) * 2], q = stats[((int64_t)img * groups + ga) * 2 + 1];
        double m = s / cnt, v = q / cnt - m * m;
        ma = (float)m; ra = (float)(1.0 / sqrt((v > 0 ? v : 0) + (double)eps));
        s = stats[((int64_t)img * groups + gb) * 2]; q = stats[((int64_t)img * groups + gb) * 2 + 1];
        m = s / cnt; v = q / cnt - m * m;
        mb = (float)m; rb = (float)(1.0 / sqrt((v > 0 ? v : 0) + (double)eps));
    }
    const float4 g = *reinterpret_cast<const float4*>(gamma + c);
    const float4 b = *reinterpret_cast<const float4*>(beta + c);
    const int64_t r0 = (int64_t)blockIdx.x * rows_per_block;
    const int64_t r1 = min(rows, r0 + rows_per_block);
#pragma unroll 4
    for (int64_t r = r0 + threadIdx.y; r < r1; r += blockDim.y) {
        const int64_t off = ((int64_t)img * rows + r) * C + c;
        float x0, x1, x2, x3;
        if (IN_F32) {
            float4 v = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(in) + off);
            x0 = v.x; x1 = v.y; x2 = v.z; x3 = v.w;
        } else {
            uint2 v = *reinterpret_cast<const uint2*>(reinterpret_cast<const act_t*>(in) + off);
            float2 a = unpack2(v.x), bb = unpack2(v.y);
            x0 = a.x; x1 = a.y; x2 = bb.x; x3 = bb.y;
        }
        x0 = (x0 - ma) * ra * g.x + b.x;
        x1 = (x1 - ma) * ra * g.y + b.y;
        x2 = (x2 - mb) * rb * g.z + b.z;
        x3 = (x3 - mb) * rb * g.w + b.w;
        if (do_silu) { x0 = ptx::silu(x0); x1 = ptx::silu(x1); x2 = ptx::silu(x2); x3 = ptx::silu(x3); }
        *reinterpret_cast<uint2*>(out + off) = make_uint2(pack2(x0, x1), pack2(x2, x3));
    }
}

static int gn_geometry(int64_t n_img, int64_t rows, int C, int groups, dim3* grid, dim3* block, int* rpb) {
    GCD_REQUIRE(C % 4 == 0 && C / 4 <= 1024, "groupnorm: C=%d unsupported", C);
    GCD_REQUIRE(groups > 0 && groups <= 64 && C % groups == 0 && (C / groups) % 2 == 0,
                "groupnorm: C=%d groups=%d unsupported (need even channels per group, <=64 groups)", C, groups);
    // ~256-thread blocks, ONE wave of them over the device's SMs (480-thread blocks at 48 registers leave 2 resident blocks =
    // 47 % occupancy and two waves)
    int bx = C / 4;
    int by = 256 / bx;
    if (by < 1) by = 1;
    if (by > 64) by = 64;
    const int threads = bx * by;
    int per_sm = 1280 / threads;              // resident blocks per SM at <= 48 registers per thread (ptxas: 40-48)
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 8) per_sm = 8;
    static const int num_sms = [] { int d = 0, n = 0; cudaGetDevice(&d); cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d); return n > 0 ? n : 132; }();
    int64_t want_blocks = (int64_t)num_sms * per_sm;
    int64_t chunks = want_blocks / (n_img > 0 ? n_img : 1);
    if (chunks < 1) chunks = 1;
    int64_t r = (rows + chunks - 1) / chunks;
    int64_t minr = (int64_t)by * 4;
    if (r < minr) r = minr;
    *rpb = (int)r;
    *grid = dim3((unsigned)((rows + r - 1) / r), (unsigned)n_img);
    *block = dim3(bx, by);
    GCD_REQUIRE(n_img <= 65535, "groupnorm: too many images (%lld)", (long long)n_img);
    return 0;
}

extern "C" int gcd_groupnorm_stats(const void* in, int in_f32, int64_t n_img, int64_t rows, int C, int groups,
                                   double* stats, void* stream) {
    dim3 grid, block;
    int rpb;
    int rc = gn_geometry(n_img, rows, C, groups, &grid, &block, &rpb);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = (size_t)block.y * (C / 2) * 2 * sizeof(double);
    GCD_REQUIRE(smem <= 48 * 1024 && (int)(block.x * block.y) >= groups, "groupnorm_stats: unsupported geometry (C=%d)", C);
    if (in_f32)
        gn_stats_kernel<true><<<grid, block, smem, st>>>(in, rows, C, C / groups, rpb, stats, groups);
    else
        gn_stats_kernel<false><<<grid, block, smem, st>>>(in, rows, C, C / groups, rpb, stats, groups);
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches++;
    return 0;
}

extern "C" int gcd_concat_channels_stats(const float* a, int Ca, const float* b, int Cb, int64_t n_img, int64_t rows,
                                         int groups, float* out, double* stats, void* stream) {
    GCD_REQUIRE(a && b && out && stats && Ca % 4 == 0 && Cb % 4 == 0, "concat_stats: channel counts must be multiples of 4");
    dim3 grid, block;
    int rpb;
    const int C = Ca + Cb;
    int rc = gn_geometry(n_img, rows, C, groups, &grid, &block, &rpb);
    if (rc) return rc;
    const size_t smem = (size_t)block.y * (C / 2) * 2 * sizeof(double);
    GCD_REQUIRE(smem <= 48 * 1024 && (int)(block.x * block.y) >= groups, "concat_stats: unsupported geometry (C=%d)", C);
    concat_stats_kernel<false><<<grid, block, smem, (cudaStream_t)stream>>>(a, Ca, b, Cb, rows, C / groups, rpb, out, stats, groups);
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches++;
    return 0;
}

extern "C" int gcd_concat_channels_stats_act(const float* a, int Ca, const float* b, int Cb, int64_t n_img, int64_t rows,
                                             int groups, void* out, double* stats, void* stream) {
    GCD_REQUIRE(a && b && out && stats && Ca % 4 == 0 && Cb % 4 == 0, "concat_stats_act: channel counts must be multiples of 4");
    dim3 grid, block;
    int rpb;
    const int C = Ca + Cb;
    int rc = gn_geometry(n_img, rows, C, groups, &grid, &block, &rpb);
    if (rc) return rc;
    const size_t smem = (size_t)block.y * (C / 2) * 2 * sizeof(double);
    GCD_REQUIRE(smem <= 48 * 1024 && (int)(block.x * block.y) >= groups, "concat_stats_act: unsupported geometry (C=%d)", C);
    concat_stats_kernel<true><<<grid, block, smem, (cudaStream_t)stream>>>(a, Ca, b, Cb, rows, C / groups, rpb, out, stats, groups);
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches++;
    return 0;
}

extern "C" int gcd_groupnorm_apply(const void* in, int in_f32, int64_t n_img, int64_t rows, int C, int groups,
                                   const double* stats, const float* gamma, const float* beta, float eps, int silu,
                                   void* out, void* stream) {
    dim3 grid, block;
    int rpb;
    int rc = gn_geometry(n_img, rows, C, groups, &grid, &block, &rpb);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (in_f32)
        gn_apply_kernel<true><<<grid, block, 0, st>>>(in, rows, C, C / groups, rpb, stats, groups, gamma, beta, eps, silu,
                                                      (act_t*)out);
    else
        gn_apply_kernel<false><<<grid, block, 0, st>>>(in, rows, C, C / groups, rpb, stats, groups, gamma, beta, eps, silu,
                                                       (act_t*)out);
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches++;
    return 0;
}

// ---------------------------------------------------------------------------------------------- LayerNorm
// One warp per row; the row (<= 2048 channels) lives in registers: mean, then centred variance (two-pass, fp32).
constexpr int LN_MAXK = 32;  // float2 per lane -> C <= 2048
template <typename OutT>     // act_t, or float for a normalised tensor that is itself a residual stream (gcd_layernorm_f32)
__global__ void layernorm_kernel(const float* __restrict__ in, int64_t rows, int C, const float* __restrict__ gamma,
                                 const float* __restrict__ beta, float eps, const float* __restrict__ add,
                                 int64_t add_rows_per, int64_t add_mod, float* __restrict__ sum_out,
                                 OutT* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int nk = C >> 6;  // float2 chunks per lane
    const float2* src = reinterpret_cast<const float2*>(in + row * C);
    const float2* ad = add ? reinterpret_cast<const float2*>(add + ((row / add_rows_per) % add_mod) * C) : nullptr;
    float2 v[LN_MAXK];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < LN_MAXK; k++) {
        if (k < nk) {
            float2 t = src[lane + 32 * k];
            if (ad) { float2 a = __ldg(&ad[lane + 32 * k]); t.x += a.x; t.y += a.y; }
            v[k] = t;
            s += t.x + t.y;
        }
    }
    if (sum_out) {
        float2* so = reinterpret_cast<float2*>(sum_out + row * C);
#pragma unroll
        for (int k = 0; k < LN_MAXK; k++)
            if (k < nk) so[lane + 32 * k] = v[k];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)C;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < LN_MAXK; k++) {
        if (k < nk) {
            float dx = v[k].x - mean, dy = v[k].y - mean;
            q += dx * dx + dy * dy;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q / (float)C + eps);
    const float2* g2 = reinterpret_cast<const float2*>(gamma);
    const float2* b2 = reinterpret_cast<const float2*>(beta);
#pragma unroll
    for (int k = 0; k < LN_MAXK; k++) {
        if (k < nk) {
            float2 g = __ldg(&g2[lane + 32 * k]), b = __ldg(&b2[lane + 32 * k]);
            const float y0 = (v[k].x - mean) * rstd * g.x + b.x, y1 = (v[k].y - mean) * rstd * g.y + b.y;
            if constexpr (sizeof(OutT) == 4) reinterpret_cast<float2*>(out + row * C)[lane + 32 * k] = make_float2(y0, y1);
            else reinterpret_cast<uint32_t*>(out + row * C)[lane + 32 * k] = pack2(y0, y1);
        }
    }
}

// Specialised version: NK float2 per lane per row, ROWS rows per warp in flight (4x the memory-level parallelism of the
// generic kernel, which measured 0.96 TB/s at C=320 — latency bound; profiles/r1_notes.md).
template <int NK, int ROWS>
__global__ void __launch_bounds__(256)
layernorm_rows_kernel(const float* __restrict__ in, int64_t rows, const float* __restrict__ gamma,
                      const float* __restrict__ beta, float eps, const float* __restrict__ add, int64_t add_rows_per,
                      int64_t add_mod, float* __restrict__ sum_out, act_t* __restrict__ out) {
    constexpr int C = NK * 64;
    const int lane = threadIdx.x & 31;
    const int64_t row0 = ((int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * ROWS;
    if (row0 >= rows) return;
    float2 v[ROWS][NK];
#pragma unroll
    for (int r = 0; r < ROWS; r++) {
        const int64_t row = row0 + r;
        if (row < rows) {
            const float2* src = reinterpret_cast<const float2*>(in + row * C);
#pragma unroll
            for (int k = 0; k < NK; k++) v[r][k] = src[lane + 32 * k];
        } else {
#pragma unroll
            for (int k = 0; k < NK; k++) v[r][k] = make_float2(0.f, 0.f);
        }
    }
    if (add) {
#pragma unroll
        for (int r = 0; r < ROWS; r++) {
            const int64_t row = row0 + r;
            if (row < rows) {
                const float2* ad = reinterpret_cast<const float2*>(add + ((row / add_rows_per) % add_mod) * C);
#pragma unroll
                for (int k = 0; k < NK; k++) { float2 a = __ldg(&ad[lane + 32 * k]); v[r][k].x += a.x; v[r][k].y += a.y; }
            }
        }
    }
    if (sum_out) {                                     // in (+ add), like the generic kernel: also written without `add`
#pragma unroll
        for (int r = 0; r < ROWS; r++) {
            const int64_t row = row0 + r;
            if (row < rows) {
                float2* so = reinterpret_cast<float2*>(sum_out + row * C);
#pragma unroll
                for (int k = 0; k < NK; k++) so[lane + 32 * k] = v[r][k];
            }
        }
    }
    float g[NK * 2], b[NK * 2];
#pragma unroll
    for (int k = 0; k < NK; k++) {
        float2 t = __ldg(reinterpret_cast<const float2*>(gamma) + lane + 32 * k);
        g[2 * k] = t.x; g[2 * k + 1] = t.y;
        t = __ldg(reinterpret_cast<const float2*>(beta) + lane + 32 * k);
        b[2 * k] = t.x; b[2 * k + 1] = t.y;
    }
#pragma unroll
    for (int r = 0; r < ROWS; r++) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < NK; k++) s += v[r][k].x + v[r][k].y;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        const float mean = s * (1.0f / C);
        float q = 0.f;
#pragma unroll
        for (int k = 0; k < NK; k++) {
            const float dx = v[r][k].x - mean, dy = v[r][k].y - mean;
            q += dx * dx + dy * dy;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
        const float rstd = rsqrtf(q * (1.0f / C) + eps);
        const int64_t row = row0 + r;
        if (row < rows) {
            uint32_t* dst = reinterpret_cast<uint32_t*>(out + row * C);
#pragma unroll
            for (int k = 0; k < NK; k++)
                dst[lane + 32 * k] = pack2((v[r][k].x - mean) * rstd * g[2 * k] + b[2 * k],
                                           (v[r][k].y - mean) * rstd * g[2 * k + 1] + b[2 * k + 1]);
        }
    }
}

template <int NK, int ROWS>
static int launch_ln(const float* in, int64_t rows, const float* gamma, const float* beta, float eps, const float* add,
                     int64_t arp, int64_t amod, float* sum_out, void* out, void* stream) {
    const int warps = 8;
    const int64_t blocks = (rows + warps * ROWS - 1) / (warps * ROWS);
    layernorm_rows_kernel<NK, ROWS><<<(unsigned)blocks, warps * 32, 0, (cudaStream_t)stream>>>(
        in, rows, gamma, beta, eps, add, arp, amod, sum_out, (act_t*)out);
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches++;
    return 0;
}

extern "C" int gcd_layernorm(const float* in, int64_t rows, int C, const float* gamma, const float* beta, float eps,
                             const float* add, int64_t add_rows_per, int64_t add_mod, float* sum_out, void* out,
                             void* stream) {
    GCD_REQUIRE(C % 64 == 0 && C <= 64 * LN_MAXK, "layernorm: C=%d must be a multiple of 64 and <= %d", C, 64 * LN_MAXK);
    GCD_REQUIRE(!add || (add_rows_per > 0 && add_mod > 0), "layernorm: bad add indexing");
    switch (C) {
        case 320: return launch_ln<5, 4>(in, rows, gamma, beta, eps, add, add_rows_per, add_mod, sum_out, out, stream);
        case 640: return launch_ln<10, 4>(in, rows, gamma, beta, eps, add, add_rows_per, add_mod, sum_out, out, stream);
        case 1280: return launch_ln<20, 2>(in, rows, gamma, beta, eps, add, add_rows_per, add_mod, sum_out, out, stream);
        default: break;
    }
    const int warps = 8;
    int64_t blocks = (rows + warps - 1) / warps;
    layernorm_kernel<act_t><<<(unsigned)blocks, warps * 32, 0, (cudaStream_t)stream>>>(in, rows, C, gamma, beta, eps, add,
                                                                                       add_rows_per, add_mod, sum_out,
                                                                                       (act_t*)out);
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches++;
    return 0;
}

// The same LayerNorm with a float32 output: the ViT's ln_pre output is the residual stream itself (open_clip
// VisionTransformer.forward: x = ln_pre(x + positional_embedding), then x = x + attn(ln_1(x)) ...), so it stays fp32.
extern "C" int gcd_layernorm_f32(const float* in, int64_t rows, int C, const float* gamma, const float* beta, float eps,
                                 const float* add, int64_t add_rows_per, int64_t add_mod, float* out, void* stream) {
    GCD_REQUIRE(C % 64 == 0 && C <= 64 * LN_MAXK, "layernorm_f32: C=%d must be a multiple of 64 and <= %d", C, 64 * LN_MAXK);
    GCD_REQUIRE(!add || (add_rows_per > 0 && add_mod > 0), "layernorm_f32: bad add indexing");
    GCD_REQUIRE(out != in, "layernorm_f32: out must not alias in");
    const int warps = 8;
    const int64_t blocks = (rows + warps - 1) / warps;
    layernorm_kernel<float><<<(unsigned)blocks, warps * 32, 0, (cudaStream_t)stream>>>(in, rows, C, gamma, beta, eps, add,
                                                                                       add_rows_per, add_mod, nullptr, out);
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches++;
    return 0;
}

// ---------------------------------------------------------------------------------------------- row softmax
// model.py:161-201 AttnBlock: softmax(q k^T / sqrt(512)) with 9216 columns; one block per row, fp32 in, act out (times
// out_scale: the VAE stores 2^15 P, so that fp16 keeps weights down to 2^-40 out of its flush-to-zero range).
__global__ void softmax_rows_kernel(const float* __restrict__ in, int cols, float scale, float out_scale, act_t* __restrict__ out) {
    __shared__ float red[32];
    const int64_t row = blockIdx.x;
    const float* src = in + row * (int64_t)cols;
    float m = -INFINITY;
    for (int j = threadIdx.x; j < cols; j += blockDim.x) m = fmaxf(m, src[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    m = red[0];
    for (int i = 1; i < (blockDim.x >> 5); i++) m = fmaxf(m, red[i]);
    __syncthreads();
    float s = 0.f;
    for (int j = threadIdx.x; j < cols; j += blockDim.x) s += __expf((src[j] - m) * scale);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    s = 0.f;
    for (int i = 0; i < (blockDim.x >> 5); i++) s += red[i];
    const float inv = out_scale / s;
    act_t* dst = out + row * (int64_t)cols;
    for (int j = threadIdx.x; j < cols; j += blockDim.x) dst[j] = f2act(__expf((src[j] - m) * scale) * inv);
}
extern "C" int gcd_softmax_rows(const float* in, int64_t rows, int cols, float scale, float out_scale, void* out, void* stream) {
    GCD_REQUIRE(rows < (1ll << 31), "softmax_rows: too many rows");
    softmax_rows_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(in, cols, scale, out_scale, (act_t*)out);
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches++;
    return 0;
}
