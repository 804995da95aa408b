// Row-level device helpers shared by the support kernels (nce_support.cu) and the fused tail kernel (nce_tail.cu):
// dtype-agnostic loads, warp reductions, the last-block mean, and the exact CUDA-core evaluation of ONE query row
// against the whole queue (the generic path, and the fallback for rows the one-sweep kernel cannot represent).
#pragma once
#include "common.cuh"
#include "sm90_ptx.cuh"

namespace moco {

__device__ __forceinline__ float load_as_float(const void* p, int dtype, size_t idx) {
    return dtype == 0 ? static_cast<const float*>(p)[idx]
                      : __bfloat162float(static_cast<const __nv_bfloat16*>(p)[idx]);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Deterministic mean over rows by the last block to finish (fixed summation order).  Returns true in every thread
// of that last block (after all other blocks' writes are visible), false elsewhere.
__device__ inline bool finish_mean(unsigned int* counter, int N, const float* loss_rows, const float* prob_rows,
                            float* loss_prob) {
    __shared__ float s_red[2][32];
    __shared__ int s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        unsigned int t = atomicAdd(counter, 1u);
        s_last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (!s_last) return false;
    __threadfence();
    float a = 0.f, b = 0.f;
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
        a += __ldcg(loss_rows + i);
        b += __ldcg(prob_rows + i);
    }
    a = warp_sum(a);
    b = warp_sum(b);
    int w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    if ((threadIdx.x & 31) == 0) { s_red[0][w] = a; s_red[1][w] = b; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float sa = 0.f, sb = 0.f;
        for (int i = 0; i < nw; ++i) { sa += s_red[0][i]; sb += s_red[1][i]; }
        loss_prob[0] = sa / (float)N;
        loss_prob[1] = sb / (float)N;
        *counter = 0u;          // re-arm for the next launch on this workspace
    }
    return true;
}

constexpr int kSimtThreads = 256;
constexpr int kSimtMaxC = 1024;

// Safe range of the one-sweep kernel's per-row sums (fixed stabiliser, see nce_sweep_sm90.cu): a row with a slice sum
// above kOnePassUnsafeSum (or NaN), or a merged sum below kOnePassUnderflow, is evaluated exactly on CUDA cores instead.
constexpr float kOnePassUnsafeSum = 1.2676506e30f;    // 2^100
constexpr float kOnePassUnderflow = 8.2718061e-25f;   // 2^-80

__device__ __forceinline__ float dot_row(const float* __restrict__ qs, const __nv_bfloat16* __restrict__ row, int C) {
    float acc = 0.f;
    if ((C & 7) == 0) {
        const uint4* r4 = reinterpret_cast<const uint4*>(row);
        for (int v = 0; v < (C >> 3); ++v) {
            uint4 u = __ldg(r4 + v);
            const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float2 f = __bfloat1622float2(h[e]);
                acc = fmaf(qs[v * 8 + e * 2], f.x, acc);
                acc = fmaf(qs[v * 8 + e * 2 + 1], f.y, acc);
            }
        }
    } else {
        for (int c = 0; c < C; ++c) acc = fmaf(qs[c], __bfloat162float(row[c]), acc);
    }
    return acc;
}


struct SimtRowSmem {
    float qs[kSimtMaxC];                 // the query row as the tensor cores see it (bf16-rounded, fp32)
    float ps[kSimtThreads];
    float red_m[kSimtThreads / 32], red_s[kSimtThreads / 32];
    float bcast;
};

// lse (log2 domain) of row `qs` against the whole queue plus the positive logit lpos (natural units, un-scaled).
// All kSimtThreads threads of the block; optional dense logits row ([K+1], column 0 = positive).
__device__ inline float simt_row_stats(SimtRowSmem& sm, float lpos, const __nv_bfloat16* __restrict__ queue, int C, int K,
                                       float inv_T, float* __restrict__ logits_row) {
    const int tid = threadIdx.x;
    const float scale2 = inv_T * kLog2e;
    const float x0 = lpos * scale2;
    float m = -INFINITY, s = 0.f;
    for (int j = tid; j < K; j += kSimtThreads) {
        float d = dot_row(sm.qs, queue + (size_t)j * C, C);
        if (logits_row) logits_row[1 + j] = d * inv_T;
        float x = d * scale2;
        if (x > m) { s *= ex2(m - x); m = x; }
        s += ex2(x - m);
    }
    float wm = warp_max(m);
    float ws_ = warp_sum(m == -INFINITY ? 0.f : s * ex2(m - wm));
    if ((tid & 31) == 0) { sm.red_m[tid >> 5] = wm; sm.red_s[tid >> 5] = ws_; }
    __syncthreads();
    if (tid == 0) {
        float M = x0;
        for (int w = 0; w < kSimtThreads / 32; ++w) M = fmaxf(M, sm.red_m[w]);
        float L = ex2(x0 - M);
        for (int w = 0; w < kSimtThreads / 32; ++w)
            if (sm.red_m[w] != -INFINITY) L += sm.red_s[w] * ex2(sm.red_m[w] - M);
        sm.bcast = M + log2f(L);
        if (logits_row) logits_row[0] = lpos * inv_T;
    }
    __syncthreads();
    return sm.bcast;
}

// acc[u] = sum_j softmax_ij queue_j[c], c = tid + u * kSimtThreads (the caller adds the positive term and scales)
__device__ inline void simt_row_grad(SimtRowSmem& sm, float lse2, const __nv_bfloat16* __restrict__ queue, int C, int K,
                                     float inv_T, float (&acc)[kSimtMaxC / kSimtThreads]) {
    const int tid = threadIdx.x;
    const float scale2 = inv_T * kLog2e;
#pragma unroll
    for (int u = 0; u < kSimtMaxC / kSimtThreads; ++u) acc[u] = 0.f;
    for (int jb = 0; jb < K; jb += kSimtThreads) {
        int j = jb + tid;
        sm.ps[tid] = (j < K) ? ex2(dot_row(sm.qs, queue + (size_t)j * C, C) * scale2 - lse2) : 0.f;
        __syncthreads();
        int jn = min(kSimtThreads, K - jb);
#pragma unroll
        for (int u = 0; u < kSimtMaxC / kSimtThreads; ++u) {
            int c = tid + u * kSimtThreads;
            if (c < C) {
                float a = acc[u];
                for (int jj = 0; jj < jn; ++jj)
                    a = fmaf(sm.ps[jj], __bfloat162float(queue[(size_t)(jb + jj) * C + c]), a);
                acc[u] = a;
            }
        }
        __syncthreads();
    }
}

}  // namespace moco
