// gcd_b200 — input frame preparation of gcd-model/scripts/infer.py: decoded uint8 frames -> u8 / 255 (fp32) -> centre crop ->
// cv2.resize(INTER_LINEAR) on the float32 image -> `* 2 - 1` -> infer.py's `(x + 1) / 2` (sgm/data/common.py:121-199,
// scripts/infer.py:137). One thread per output pixel, all frames of a group in one launch.
//
// The taps follow OpenCV's resize for float32 images (imgproc/src/resize.cpp, resizeGeneric_ with HResizeLinear /
// VResizeLinear), not torch's upsample_bilinear2d (render.cu's `bilin`): the source coordinate is rounded to fp32 before the
// floor, the fraction is taken in fp32 and both borders clamp the index with fraction 0. Products and sums are separate fp32
// roundings (no FMA contraction), horizontal pass first.
#include "common.cuh"
#include "../../include/gcd_b200.h"
#include <atomic>
#include <math.h>
extern std::atomic<int64_t> g_launches;

namespace {
constexpr int FT = 256;

struct Tap { int i0, i1; float w0, w1; };

// cv2 INTER_LINEAR tap of output index d: fx = (float)((d + 0.5) * scale - 0.5), sx = floor(fx), fx -= sx; sx < 0 -> (0, f 0),
// sx >= n - 1 -> (n - 1, f 0); weights (1 - fx, fx) in fp32.
__device__ __forceinline__ Tap cv_tap(int d, int n, double scale) {
    float fx = (float)(((double)d + 0.5) * scale - 0.5);
    int sx = (int)floorf(fx);
    fx = __fsub_rn(fx, (float)sx);
    if (sx < 0) { sx = 0; fx = 0.f; }
    if (sx >= n - 1) { sx = n - 1; fx = 0.f; }
    Tap t;
    t.i0 = sx;
    t.i1 = min(sx + 1, n - 1);
    t.w0 = __fsub_rn(1.f, fx);
    t.w1 = fx;
    return t;
}

struct Params {
    const uint8_t* in;
    int H, W, C;              // decoded frame size and channels (3 or 4)
    int y0, x0, ch, cw;       // crop box
    int Ho, Wo;               // output size
    int map[3];               // output channel c reads input channel map[c]
    double sy, sx;            // ch / Ho, cw / Wo
    const int32_t* out_frame; // output frame of input frame f, or NULL (f)
    float* out;
};

__device__ __forceinline__ float u8f(uint8_t v) { return __fdiv_rn((float)v, 255.0f); }

__global__ void __launch_bounds__(FT) frames_prepare_kernel(Params p) {
    const int f = blockIdx.y;
    const int64_t i = (int64_t)blockIdx.x * FT + threadIdx.x;
    if (i >= (int64_t)p.Ho * p.Wo) return;
    const int oy = (int)(i / p.Wo), ox = (int)(i % p.Wo);
    const uint8_t* src = p.in + (int64_t)f * p.H * p.W * p.C;
    float v[3];
    if (p.Ho == p.ch && p.Wo == p.cw) {                      // no resize: the cropped pixel itself
        const uint8_t* q = src + ((int64_t)(p.y0 + oy) * p.W + p.x0 + ox) * p.C;
#pragma unroll
        for (int c = 0; c < 3; c++) v[c] = u8f(q[p.map[c]]);
    } else {
        const Tap ty = cv_tap(oy, p.ch, p.sy), tx = cv_tap(ox, p.cw, p.sx);
        const uint8_t* r0 = src + (int64_t)(p.y0 + ty.i0) * p.W * p.C;
        const uint8_t* r1 = src + (int64_t)(p.y0 + ty.i1) * p.W * p.C;
        const int c0 = (p.x0 + tx.i0) * p.C, c1 = (p.x0 + tx.i1) * p.C;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const int m = p.map[c];
            const float h0 = __fadd_rn(__fmul_rn(u8f(r0[c0 + m]), tx.w0), __fmul_rn(u8f(r0[c1 + m]), tx.w1));
            const float h1 = __fadd_rn(__fmul_rn(u8f(r1[c0 + m]), tx.w0), __fmul_rn(u8f(r1[c1 + m]), tx.w1));
            v[c] = __fadd_rn(__fmul_rn(h0, ty.w0), __fmul_rn(h1, ty.w1));
        }
    }
    const int fo = p.out_frame ? p.out_frame[f] : f;
    float* o = p.out + (int64_t)fo * 3 * p.Ho * p.Wo + i;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        // process_image's `* 2 - 1`, then infer.py's `(x + 1) / 2`: not the identity below 0.5 in fp32
        const float x = __fsub_rn(__fmul_rn(v[c], 2.f), 1.f);
        o[(int64_t)c * p.Ho * p.Wo] = __fdiv_rn(__fadd_rn(x, 1.f), 2.f);
    }
}
}  // namespace

extern "C" int gcd_frames_prepare(const uint8_t* in, int n, int H, int W, int C, const int32_t* channel_map, int y0, int x0,
                                  int ch, int cw, int Ho, int Wo, const int32_t* out_frame, float* out, void* stream) {
    GCD_REQUIRE(in && channel_map && out && n > 0, "frames_prepare: null pointer or no frames");
    GCD_REQUIRE(n <= 65535, "frames_prepare: at most 65535 frames per call");
    GCD_REQUIRE(H > 0 && W > 0 && (C == 3 || C == 4) && Ho > 0 && Wo > 0, "frames_prepare: bad sizes (C must be 3 or 4)");
    GCD_REQUIRE(y0 >= 0 && x0 >= 0 && ch > 0 && cw > 0 && y0 + ch <= H && x0 + cw <= W,
                "frames_prepare: crop box (%d, %d, %d, %d) outside the %d x %d frame", y0, x0, ch, cw, H, W);
    Params p;
    p.in = in; p.H = H; p.W = W; p.C = C;
    p.y0 = y0; p.x0 = x0; p.ch = ch; p.cw = cw; p.Ho = Ho; p.Wo = Wo;
    for (int c = 0; c < 3; c++) {
        GCD_REQUIRE(channel_map[c] >= 0 && channel_map[c] < 3, "frames_prepare: channel map entries must be 0..2");
        p.map[c] = channel_map[c];
    }
    p.sy = (double)ch / Ho;
    p.sx = (double)cw / Wo;
    p.out_frame = out_frame;
    p.out = out;
    const dim3 grid((unsigned)(((int64_t)Ho * Wo + FT - 1) / FT), n);
    frames_prepare_kernel<<<grid, FT, 0, (cudaStream_t)stream>>>(p);
    GCD_CUDA_CHECK(cudaGetLastError());
    g_launches += 1;
    return 0;
}
