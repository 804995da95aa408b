// Microbenchmark: per-SM throughput of the exp2 paths the NCE epilogue can use (H100).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/mufu_bench tools/mufu_bench.cu && /tmp/mufu_bench
#include <cstdio>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

__device__ __forceinline__ float ex2f(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ unsigned ex2h2(unsigned x) { unsigned y; asm("ex2.approx.f16x2 %0, %1;" : "=r"(y) : "r"(x)); return y; }
__device__ __forceinline__ unsigned ex2b2(unsigned x) { unsigned y; asm("ex2.approx.ftz.bf16x2 %0, %1;" : "=r"(y) : "r"(x)); return y; }

template <int MODE>
__global__ void k(float* out, int iters, float seed) {
    float a[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = seed + j * 0.01f + threadIdx.x * 1e-4f;
    float acc = 0.f;
    unsigned hacc = 0;
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (MODE == 0) {                      // MUFU.EX2 only (independent chains)
                a[j] = ex2f(a[j]) - 1.0f;
            } else if (MODE == 1) {               // the epilogue's element: FFMA -> EX2 -> FADD
                acc += ex2f(fmaf(a[j], 1.0001f, -0.5f));
                a[j] += 1e-6f;
            } else if (MODE == 2) {               // packed f16x2 ex2: two exponentials per MUFU op
                unsigned v = __float_as_uint(a[j]);
                hacc ^= ex2h2(v);
                a[j] += 1e-6f;
            } else if (MODE == 3) {               // packed bf16x2
                unsigned v = __float_as_uint(a[j]);
                hacc ^= ex2b2(v);
                a[j] += 1e-6f;
            } else if (MODE == 4) {               // polynomial exp2 on the FMA pipe (degree 4, Cody-Waite)
                float x = a[j];
                float fl = floorf(x);
                float f = x - fl;
                float p = fmaf(f, 0.0135557f, 0.0520324f);
                p = fmaf(p, f, 0.2413793f);
                p = fmaf(p, f, 0.6930580f);
                p = fmaf(p, f, 1.0f);
                acc += __uint_as_float(__float_as_uint(p) + ((int)fl << 23));
                a[j] += 1e-6f;
            }
        }
    }
    float r = acc + __uint_as_float(hacc);
#pragma unroll
    for (int j = 0; j < 8; ++j) r += a[j];
    out[blockIdx.x * blockDim.x + threadIdx.x] = r;
}

template <int MODE>
void run(const char* name, int threads) {
    int sms = 132, iters = 4096;
    float* out;
    cudaMalloc(&out, sizeof(float) * sms * threads);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    k<MODE><<<sms, threads>>>(out, iters, -3.0f);
    cudaDeviceSynchronize();
    cudaEventRecord(e0);
    k<MODE><<<sms, threads>>>(out, iters, -3.0f);
    cudaEventRecord(e1);
    cudaDeviceSynchronize();
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    int clk_khz; cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
    double ops = (double)sms * threads * iters * 8;
    double per_clk_sm = ops / (ms * 1e-3) / (clk_khz * 1e3) / sms;
    printf("%-34s threads=%4d  %.3f ms  %.2f elem/clk/SM (at nominal %d MHz)  %.2f Gelem/s\n", name, threads, ms,
           per_clk_sm, clk_khz / 1000, ops / (ms * 1e-3) / 1e9);
    cudaFree(out);
}

int main() {
    for (int threads : {256, 512, 1024}) {
        run<0>("ex2.approx.ftz.f32 only", threads);
        run<1>("ffma + ex2.f32 + fadd", threads);
        run<2>("ex2.approx.f16x2 (ops, x2 elems)", threads);
        run<3>("ex2.approx.ftz.bf16x2 (ops, x2 elems)", threads);
        run<4>("poly exp2 on FMA pipe", threads);
    }
    return 0;
}
