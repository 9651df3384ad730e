// gcd_b200 — point-cloud view synthesis of the evaluation clips (Kubric-4D / ParDom-4D): the conditioning video, the target video and
// the reprojection baseline that gcd-model/sgm/data/kubric_arbit.py:410-563 (synth_src_dst_rgb) and pardom_arbit.py:585-738
// (synth_rgb) render per frame from the stored clouds with geometry.py:242-444 (project_points_to_pixels, spreaded_index_add,
// blur_into_black) followed by a bilinear resize and `* 2 - 1`.
//
// Every render of a call (any number of frames, cameras, blur sizes) goes through the same three launches:
//   render_depth_kernel   one thread per (render, point): project in fp64, the maximum depth of the valid points per render;
//   render_splat_kernel   one thread per (render, point): weight exp(-depth_norm * strength), fp64 atomics of
//                         (w r, w g, w b, w) into the [H*W, 4] accumulator at the centre pixel and the spread offsets (x 0.02);
//   render_image_kernel   one block per 32x16 tile of the model-size output: normalise / clamp / black mask, the masked
//                         Gaussian leak (separable, reflect border), the 3x3 sigma 0.6 blur, the bilinear resize, `* 2 - 1`.
// The weights span e^-512..e^512 (Kubric) so the accumulator is fp64 like the reference's; H100 has native fp64 atomics.
#include "common.cuh"
#include "../../include/gcd_b200.h"
#include <atomic>
#include <math.h>
#include <vector>
extern std::atomic<int64_t> g_launches;

namespace {
constexpr int PT = 256;                       // point-pass threads per block
constexpr int OTX = 32, OTY = 16, IT = 256;   // image pass: output tile and threads
constexpr int MAX_K = 31;

struct Proj { bool ok; int ix, iy; double depth; };

// geometry.py:231-284: world_to_camera, K x / (K x)_z, uv_int = (int32)(uv + 0.5) (truncation toward zero, so uv in (-1.5, -0.5)
// lands in column / row 0), valid if inside the image and depth > 0.1. Non-finite coordinates are dropped (torch's CPU cast turns
// a NaN uv into INT_MIN; its CUDA cast gives 0 — DESIGN.md §3 "render").
__device__ __forceinline__ Proj project(const __half* __restrict__ xyz, const double* __restrict__ cam, int H, int W) {
    const double x = __half2float(xyz[0]) - cam[18], y = __half2float(xyz[1]) - cam[19], z = __half2float(xyz[2]) - cam[20];
    const double* R = cam + 9;                           // xyz_camera = (xyz - t) @ R
    const double cx = x * R[0] + y * R[3] + z * R[6];
    const double cy = x * R[1] + y * R[4] + z * R[7];
    const double cz = x * R[2] + y * R[5] + z * R[8];
    const double* K = cam;
    const double u = K[0] * cx + K[1] * cy + K[2] * cz;
    const double v = K[3] * cx + K[4] * cy + K[5] * cz;
    const double w = K[6] * cx + K[7] * cy + K[8] * cz;
    const double uu = u / w + 0.5, vv = v / w + 0.5;
    Proj p;
    p.ok = uu > -1.0 && uu < (double)W && vv > -1.0 && vv < (double)H && cz > 0.1;   // false for NaN
    p.ix = p.ok ? (int)uu : 0;
    p.iy = p.ok ? (int)vv : 0;
    p.depth = cz;
    return p;
}

__global__ void __launch_bounds__(PT)
render_depth_kernel(const __half* __restrict__ xyz, int64_t P, const int* __restrict__ desc, const double* __restrict__ cams,
                    int H, int W, unsigned long long* __restrict__ maxd) {
    const int r = blockIdx.y;
    const int f = desc[r * 4], n = desc[r * 4 + 2];
    const int64_t i = (int64_t)blockIdx.x * PT + threadIdx.x;
    double d = 0.0;
    if (i < n) {
        const Proj p = project(xyz + ((int64_t)f * P + desc[r * 4 + 1] + i) * 3, cams + r * 24, H, W);
        if (p.ok) d = p.depth;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d = fmax(d, __shfl_xor_sync(0xffffffffu, d, o));
    // positive doubles order like their bit patterns
    if ((threadIdx.x & 31) == 0 && d > 0.0) atomicMax(maxd + r, (unsigned long long)__double_as_longlong(d));
}

__global__ void __launch_bounds__(PT)
render_splat_kernel(const __half* __restrict__ xyz, const uint8_t* __restrict__ rgb, const uint8_t* __restrict__ segm,
                    const float* __restrict__ palette, int64_t P, const int* __restrict__ desc, const double* __restrict__ cams,
                    int H, int W, int spread, const unsigned long long* __restrict__ maxd, double* __restrict__ acc) {
    const int r = blockIdx.y;
    const int f = desc[r * 4], n = desc[r * 4 + 2];
    const int64_t i = (int64_t)blockIdx.x * PT + threadIdx.x;
    if (i >= n) return;
    const int64_t pi = (int64_t)f * P + desc[r * 4 + 1] + i;
    const double* cam = cams + r * 24;
    const Proj p = project(xyz + pi * 3, cam, H, W);
    if (!p.ok) return;
    double m = __longlong_as_double((long long)maxd[r]), d = p.depth, strength = 512.0;
    if (m >= 64.0) {                        // ParDom: sqrt, clamp to 32 (monotone, so the max maps through)
        strength = 256.0;
        d = fmin(fmax(sqrt(d), 0.0), 32.0);
        m = fmin(fmax(sqrt(m), 0.0), 32.0);
    }
    const double dn = __dadd_rn(__dmul_rn(__ddiv_rn(d, m), 2.0), -1.0);
    const double wgt = exp(__dmul_rn(-dn, strength));
    // colour: (u8 / 255.0) in fp32; ParDom segm blends (1 - a) rgb + a palette[id] in fp32 (pardom_arbit.py:638-665)
    float c[3];
    const float a = (float)cam[21], oma = (float)(1.0 - cam[21]);
#pragma unroll
    for (int k = 0; k < 3; k++) {
        c[k] = __fdiv_rn((float)rgb[pi * 3 + k], 255.0f);
        if (segm) c[k] = __fadd_rn(__fmul_rn(oma, c[k]), __fmul_rn(a, palette[segm[pi] * 3 + k]));
    }
    const double v[4] = {(double)c[0] * wgt, (double)c[1] * wgt, (double)c[2] * wgt, wgt};
    double* base = acc + (int64_t)r * H * W * 4;
    double* px = base + ((int64_t)p.iy * W + p.ix) * 4;
#pragma unroll
    for (int k = 0; k < 4; k++) atomicAdd(px + k, v[k]);
    const int lo = -(spread / 2), hi = (spread + 1) / 2;   // spreaded_index_add's offsets (geometry.py:375-399)
    for (int dx = lo; dx <= hi; dx++)
        for (int dy = lo; dy <= hi; dy++) {
            if (dx == 0 && dy == 0) continue;
            const int x = p.ix + dx, y = p.iy + dy;
            if (x < 0 || x >= W || y < 0 || y >= H) continue;
            double* q = base + ((int64_t)y * W + x) * 4;
#pragma unroll
            for (int k = 0; k < 4; k++) atomicAdd(q + k, v[k] * 0.02);
        }
}

__device__ __forceinline__ int reflect(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * (n - 1) - i : i); }

// torchvision _get_gaussian_kernel1d in fp64: linspace(-h, h, k), exp(-0.5 (x / sigma)^2), normalised
__device__ void gauss_taps(double* t, int k, double sigma) {
    double s = 0.0;
    for (int j = 0; j < k; j++) {
        const double x = (double)(j - k / 2) / sigma;
        t[j] = exp(-0.5 * (x * x));
        s += t[j];
    }
    for (int j = 0; j < k; j++) t[j] /= s;
}

struct Src { int i0, i1; double l1; };
// upsample_bilinear2d, align_corners = False, scale = in / out in fp64
__host__ __device__ __forceinline__ Src bilin(int o, int n_in, double scale) {
    double s = scale * (o + 0.5) - 0.5;
    if (s < 0.0) s = 0.0;
    Src r;
    r.i0 = (int)s;
    r.i1 = r.i0 + (r.i0 < n_in - 1 ? 1 : 0);
    r.l1 = s - r.i0;
    return r;
}

struct Extent { int r3lo, r3hi, r2lo, r2hi, r1lo, r1hi; };
__host__ __device__ __forceinline__ Extent extent(int o0, int o_last, int n_in, double scale, int h) {
    Extent e;
    e.r3lo = bilin(o0, n_in, scale).i0;
    e.r3hi = bilin(o_last, n_in, scale).i1;
    e.r2lo = max(0, e.r3lo - 1); e.r2hi = min(n_in - 1, e.r3hi + 1);
    e.r1lo = max(0, e.r2lo - h); e.r1hi = min(n_in - 1, e.r2hi + h);
    return e;
}

__global__ void __launch_bounds__(IT)
render_image_kernel(const double* __restrict__ acc, const int* __restrict__ desc, int H, int W, int Hp, int Wp,
                    float* __restrict__ out) {
    extern __shared__ double smem[];
    __shared__ double tk[MAX_K], t3[3];
    const int r = blockIdx.z, k = desc[r * 4 + 3], h = k / 2;
    const double sy = (double)H / Hp, sx = (double)W / Wp;
    const int oy0 = blockIdx.y * OTY, ox0 = blockIdx.x * OTX;
    const int oy1 = min(oy0 + OTY, Hp) - 1, ox1 = min(ox0 + OTX, Wp) - 1;
    const Extent ey = extent(oy0, oy1, H, sy, h), ex = extent(ox0, ox1, W, sx, h);
    const int n1y = ey.r1hi - ey.r1lo + 1, n1x = ex.r1hi - ex.r1lo + 1;
    const int n2y = ey.r2hi - ey.r2lo + 1, n2x = ex.r2hi - ex.r2lo + 1;
    if (threadIdx.x == 0) gauss_taps(tk, k, k / 4.0);
    if (threadIdx.x == 32) gauss_taps(t3, 3, 0.6);
    float4* s1 = reinterpret_cast<float4*>(smem);                       // [n1y][n1x] normalised image, borrow mask
    double4* hb = reinterpret_cast<double4*>(s1 + ((n1y * n1x + 1) & ~1)); // [n1y][n2x] horizontal blur
    double* s2 = reinterpret_cast<double*>(hb + n1y * n2x);               // [n2y][n2x][3] after the leak
    const double* pa = acc + (int64_t)r * H * W * 4;

    // project_points_to_pixels' normalise: weight <= 0 -> -1, divide, clamp to [0, 1], float32; black = channel sum == 0
    for (int i = threadIdx.x; i < n1y * n1x; i += IT) {
        const int y = ey.r1lo + i / n1x, x = ex.r1lo + i % n1x;
        const double4 q = *reinterpret_cast<const double4*>(pa + ((int64_t)y * W + x) * 4);
        const double w = q.w <= 0.0 ? -1.0 : q.w;
        const float c0 = (float)fmin(fmax(q.x / w, 0.0), 1.0), c1 = (float)fmin(fmax(q.y / w, 0.0), 1.0),
                    c2 = (float)fmin(fmax(q.z / w, 0.0), 1.0);
        s1[i] = make_float4(c0, c1, c2, (c0 + c1 + c2 == 0.0f) ? 0.f : 1.f);
    }
    __syncthreads();
    // gaussian_blur_masked_vectorized: blur of the image and of the borrow mask, reflect border (rows r1, columns r2)
    for (int i = threadIdx.x; i < n1y * n2x; i += IT) {
        const int ly = i / n2x, x = ex.r2lo + i % n2x;
        double4 s = make_double4(0, 0, 0, 0);
        for (int j = -h; j <= h; j++) {
            const float4 v = s1[ly * n1x + reflect(x + j, W) - ex.r1lo];
            const double t = tk[j + h];
            s.x += t * v.x; s.y += t * v.y; s.z += t * v.z; s.w += t * v.w;
        }
        hb[i] = s;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n2y * n2x; i += IT) {
        const int y = ey.r2lo + i / n2x, lx = i % n2x, x = ex.r2lo + lx;
        const float4 c = s1[(y - ey.r1lo) * n1x + x - ex.r1lo];
        double* o = s2 + i * 3;
        if (c.w != 0.f) {                                                  // not black: kept as is
            o[0] = c.x; o[1] = c.y; o[2] = c.z;
        } else {                                                           // black: blur(img) / clamp(blur(mask), 1e-7)
            double4 s = make_double4(0, 0, 0, 0);
            for (int j = -h; j <= h; j++) {
                const double4 v = hb[(reflect(y + j, H) - ey.r1lo) * n2x + lx];
                const double t = tk[j + h];
                s.x += t * v.x; s.y += t * v.y; s.z += t * v.z; s.w += t * v.w;
            }
            const double m = fmax(s.w, 1e-7);
            o[0] = s.x / m; o[1] = s.y / m; o[2] = s.z / m;
        }
    }
    __syncthreads();
    // 3x3 sigma 0.6 blur (reflect) evaluated at the bilinear taps, then `* 2 - 1`
    float* po = out + (int64_t)r * 3 * Hp * Wp;
    for (int i = threadIdx.x; i < OTY * OTX; i += IT) {
        const int oy = oy0 + i / OTX, ox = ox0 + i % OTX;
        if (oy >= Hp || ox >= Wp) continue;
        const Src by = bilin(oy, H, sy), bx = bilin(ox, W, sx);
        double v[2][2][3];
#pragma unroll
        for (int a = 0; a < 2; a++)
#pragma unroll
            for (int b = 0; b < 2; b++) {
                const int yy = a ? by.i1 : by.i0, xx = b ? bx.i1 : bx.i0;
                double s[3] = {0, 0, 0};
#pragma unroll
                for (int dy = -1; dy <= 1; dy++)
#pragma unroll
                    for (int dx = -1; dx <= 1; dx++) {
                        const double t = t3[dy + 1] * t3[dx + 1];
                        const double* q = s2 + ((reflect(yy + dy, H) - ey.r2lo) * n2x + reflect(xx + dx, W) - ex.r2lo) * 3;
                        s[0] += t * q[0]; s[1] += t * q[1]; s[2] += t * q[2];
                    }
                v[a][b][0] = s[0]; v[a][b][1] = s[1]; v[a][b][2] = s[2];
            }
        const double h1 = by.l1, h0 = 1.0 - h1, w1 = bx.l1, w0 = 1.0 - w1;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const double y = h0 * (w0 * v[0][0][c] + w1 * v[0][1][c]) + h1 * (w0 * v[1][0][c] + w1 * v[1][1][c]);
            po[((int64_t)c * Hp + oy) * Wp + ox] = (float)(y * 2.0 - 1.0);
        }
    }
}

size_t image_smem(int H, int W, int Hp, int Wp, int kmax) {
    const int h = kmax / 2;
    size_t best = 0;
    for (int oy0 = 0; oy0 < Hp; oy0 += OTY)
        for (int ox0 = 0; ox0 < Wp; ox0 += OTX) {
            const Extent ey = extent(oy0, std::min(oy0 + OTY, Hp) - 1, H, (double)H / Hp, h);
            const Extent ex = extent(ox0, std::min(ox0 + OTX, Wp) - 1, W, (double)W / Wp, h);
            const size_t n1 = (size_t)(ey.r1hi - ey.r1lo + 1) * (ex.r1hi - ex.r1lo + 1);
            const size_t n1h = (size_t)(ey.r1hi - ey.r1lo + 1) * (ex.r2hi - ex.r2lo + 1);
            const size_t n2 = (size_t)(ey.r2hi - ey.r2lo + 1) * (ex.r2hi - ex.r2lo + 1);
            best = std::max(best, ((n1 + 1) & ~(size_t)1) * 16 + n1h * 32 + n2 * 24);
        }
    return best;
}
}  // namespace

extern "C" int gcd_render_views(const void* xyz, const uint8_t* rgb, const uint8_t* segm, const float* palette, int64_t P, int R,
                                const int32_t* desc_host, const int32_t* desc, const double* cams, int H, int W, int Hp, int Wp,
                                int spread_radius, double* acc, double* maxd, float* out, void* stream) {
    GCD_REQUIRE(xyz && rgb && desc_host && desc && cams && acc && maxd && out && R > 0 && P > 0,
                "render_views: null pointer or empty batch");
    GCD_REQUIRE(!segm == !palette, "render_views: segm and palette go together");
    GCD_REQUIRE(H > 0 && W > 0 && Hp > 0 && Wp > 0 && spread_radius >= 0 && spread_radius <= 8, "render_views: bad sizes");
    GCD_REQUIRE(R <= 65535, "render_views: at most 65535 renders per call");
    int nmax = 0, kmax = 1;
    for (int r = 0; r < R; r++) {
        const int32_t* d = desc_host + r * 4;
        GCD_REQUIRE(d[0] >= 0 && d[1] >= 0 && d[2] > 0 && (int64_t)d[1] + d[2] <= P, "render_views: render %d point range", r);
        GCD_REQUIRE(d[3] >= 1 && d[3] <= MAX_K && (d[3] & 1), "render_views: render %d blur kernel must be odd, 1..%d", r, MAX_K);
        GCD_REQUIRE(d[3] / 2 < H && d[3] / 2 < W, "render_views: reflect padding needs the blur radius below the render size");
        nmax = std::max(nmax, (int)d[2]);
        kmax = std::max(kmax, (int)d[3]);
    }
    const size_t smem = image_smem(H, W, Hp, Wp, kmax);
    GCD_REQUIRE(smem <= 227 * 1024, "render_views: render / frame size ratio too large for one tile (%zu B shared)", smem);
    cudaStream_t st = (cudaStream_t)stream;
    GCD_CUDA_CHECK(cudaMemsetAsync(acc, 0, (size_t)R * H * W * 4 * sizeof(double), st));
    GCD_CUDA_CHECK(cudaMemsetAsync(maxd, 0, (size_t)R * sizeof(double), st));
    const dim3 pgrid((nmax + PT - 1) / PT, R);
    const __half* x = (const __half*)xyz;
    render_depth_kernel<<<pgrid, PT, 0, st>>>(x, P, desc, cams, H, W, (unsigned long long*)maxd);
    GCD_CUDA_CHECK(cudaGetLastError());
    render_splat_kernel<<<pgrid, PT, 0, st>>>(x, rgb, segm, palette, P, desc, cams, H, W, spread_radius,
                                              (const unsigned long long*)maxd, acc);
    GCD_CUDA_CHECK(cudaGetLastError());
    GCD_CUDA_CHECK(cudaFuncSetAttribute(render_image_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const dim3 igrid((Wp + OTX - 1) / OTX, (Hp + OTY - 1) / OTY, R);
    render_image_kernel<<<igrid, IT, smem, st>>>(acc, desc, H, W, Hp, Wp, out);
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches += 3;
    return 0;
}
