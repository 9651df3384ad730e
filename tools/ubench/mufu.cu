// Micro-benchmark: MUFU ex2 throughput per SM for f32, f16x2 and bf16x2 operands (is the packed form 2 exps per lane-op?).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench/mufu tools/ubench/mufu.cu
#include <cstdio>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
template <int MODE>
__global__ void k(float* out, int iters, float seed) {
    float a0 = seed + threadIdx.x * 1e-6f, a1 = a0 + 0.1f, a2 = a0 + 0.2f, a3 = a0 + 0.3f;
    unsigned h0 = 0x38003800u + threadIdx.x, h1 = h0 + 1, h2 = h0 + 2, h3 = h0 + 3;
    for (int i = 0; i < iters; i++) {
        if (MODE == 0) {
            asm volatile("ex2.approx.ftz.f32 %0, %0;" : "+f"(a0)); asm volatile("ex2.approx.ftz.f32 %0, %0;" : "+f"(a1));
            asm volatile("ex2.approx.ftz.f32 %0, %0;" : "+f"(a2)); asm volatile("ex2.approx.ftz.f32 %0, %0;" : "+f"(a3));
        } else if (MODE == 1) {
            asm volatile("ex2.approx.f16x2 %0, %0;" : "+r"(h0)); asm volatile("ex2.approx.f16x2 %0, %0;" : "+r"(h1));
            asm volatile("ex2.approx.f16x2 %0, %0;" : "+r"(h2)); asm volatile("ex2.approx.f16x2 %0, %0;" : "+r"(h3));
        } else {
            asm volatile("ex2.approx.ftz.bf16x2 %0, %0;" : "+r"(h0)); asm volatile("ex2.approx.ftz.bf16x2 %0, %0;" : "+r"(h1));
            asm volatile("ex2.approx.ftz.bf16x2 %0, %0;" : "+r"(h2)); asm volatile("ex2.approx.ftz.bf16x2 %0, %0;" : "+r"(h3));
        }
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + __uint_as_float(h0 ^ h1 ^ h2 ^ h3);
}
int main() {
    float* out; cudaMalloc(&out, 132 * 8 * 1024 * 4);
    int clk; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    const int iters = 20000, blocks = 132 * 2, threads = 1024;
    const char* names[3] = {"ex2.f32", "ex2.f16x2", "ex2.bf16x2"};
    for (int m = 0; m < 3; m++) {
        cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
        for (int rep = 0; rep < 2; rep++) {
            cudaEventRecord(e0);
            if (m == 0) k<0><<<blocks, threads>>>(out, iters, 0.5f);
            else if (m == 1) k<1><<<blocks, threads>>>(out, iters, 0.5f);
            else k<2><<<blocks, threads>>>(out, iters, 0.5f);
            cudaEventRecord(e1); cudaEventSynchronize(e1);
        }
        float ms; cudaEventElapsedTime(&ms, e0, e1);
        double instr = (double)blocks * threads * iters * 4;
        printf("%-10s %.3f ms  %.2f lane-instr/ns chip = %.1f lane-instr/clk/SM at max clock %d MHz (x2 values for packed)\n", names[m], ms,
               instr / (ms * 1e6), instr / (ms * 1e-3) / 132 / (clk * 1e3), clk / 1000);
    }
    printf("err %s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
