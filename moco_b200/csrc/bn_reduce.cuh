// The reduction pieces of the training BatchNorm's statistics (bn_nhwc.cu: bn_stats_kernel), shared with the 1x1
// convolution whose epilogue takes the same statistics (conv1x1_sm90.cu): both add the same values in the same order,
// so the two give bit-identical results on the same activations.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace moco {

constexpr int kBnThreads = 256;
constexpr int kBnSlab = 64;                          // channels per reduction CTA
constexpr int kBnLanes = kBnSlab / 8;                // 16-byte vectors per slab row
constexpr int kBnRows = kBnThreads / kBnLanes;       // rows per pass
// (16-byte loads in flight per thread, resident CTAs per SM) of the statistics kernel; its row plan (bn_stats_plan)
constexpr int kBnStatsUnroll = 8, kBnStatsCtas = 2;
// the same of the backward reduction kernel; its row plan (bn_bwd_reduce_plan)
constexpr int kBnBwdReduceUnroll = 4, kBnBwdReduceCtas = 2;

// the barrier of the kBnThreads threads that reduce: the whole CTA unless the caller passes its own
struct CtaSync {
    __device__ __forceinline__ void operator()() const { __syncthreads(); }
};

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float2 t = __bfloat1622float2(h[k]);
        f[2 * k] = t.x;
        f[2 * k + 1] = t.y;
    }
}

// 8 mask bits of one vector of y, from the bf16 values as stored (a positive value that rounds to zero is off)
__device__ __forceinline__ unsigned int relu_bits(const uint4& y) {
    float r[8];
    unpack8(y, r);
    unsigned int b = 0u;
#pragma unroll
    for (int k = 0; k < 8; ++k) b |= (r[k] > 0.f ? 1u : 0u) << k;
    return b;
}

// Sum the 8 * S per-thread accumulators (S per-channel sums of 8 channels) over the CTA's 32 row groups.  Returns, in
// threads j < 64 * S, element j of the CTA partial: j = v * 8S + k with v = 16-byte lane (8 channels), k < 8 the first
// sum, 8 <= k < 16 the second, 16 <= k < 24 the third.  Each element is added in the same order whatever S is.
template <int S, typename Sync = CtaSync>
__device__ __forceinline__ float slab_reduce(float (&acc)[8 * S], float* red /*[8 * 64S]*/, Sync sync = Sync()) {
    constexpr int P = S * kBnSlab;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 8 * S; ++k) {
        acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], 8);
        acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], 16);
    }
    if (lane < 8) {
#pragma unroll
        for (int k = 0; k < 8 * S; ++k) red[warp * P + lane * 8 * S + k] = acc[k];
    }
    sync();
    float t = 0.f;
    if (threadIdx.x < P) {
#pragma unroll
        for (int w = 0; w < kBnThreads / 32; ++w) t += red[w * P + threadIdx.x];
    }
    return t;
}

// Publishes this CTA's partial (64S floats), and in the last CTA of the slab to arrive returns true with the slab
// totals in tot[64S] (same element order as slab_reduce).  The R partials are added in a fixed order: warp w takes
// partials w, w + 8, ... (lane l owns floats 4l .. 4l+3 of each 128-float chunk, one coalesced 512-byte read per
// partial and chunk, 16 reads in flight), then the 8 warps' sums are added in warp order.
template <int S, typename Sync = CtaSync>
__device__ __forceinline__ bool slab_finish(float part, float* partial, unsigned int* counter, int slab, int r, int R,
                                            double* tot /*[8 * 64S] shared*/, int* flag /*shared*/, Sync sync = Sync()) {
    constexpr int P = S * kBnSlab;
    float* mine = partial + ((size_t)slab * R + r) * P;
    if (threadIdx.x < P) mine[threadIdx.x] = part;
    __threadfence();
    sync();
    if (threadIdx.x == 0) {
        const unsigned int ticket = atomicAdd(counter, 1u);
        *flag = (ticket == (unsigned int)(R - 1));
    }
    sync();
    if (!*flag) return false;
    __threadfence();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float4* base = reinterpret_cast<const float4*>(partial + (size_t)slab * R * P);
    for (int c4 = lane; c4 < P / 4; c4 += 32) {
        double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
        constexpr int kBatch = 16;
        for (int q0 = warp; q0 < R; q0 += 8 * kBatch) {
            float4 v[kBatch];
#pragma unroll
            for (int t = 0; t < kBatch; ++t) {
                const int q = q0 + 8 * t;
                v[t] = (q < R) ? __ldcg(base + (size_t)q * (P / 4) + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int t = 0; t < kBatch; ++t) { s0 += v[t].x; s1 += v[t].y; s2 += v[t].z; s3 += v[t].w; }
        }
        double* mine_tot = tot + warp * P + c4 * 4;
        mine_tot[0] = s0; mine_tot[1] = s1; mine_tot[2] = s2; mine_tot[3] = s3;
    }
    sync();
    if (threadIdx.x < P) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < 8; ++w) t += tot[w * P + threadIdx.x];
        __syncwarp();
        tot[threadIdx.x] = t;                        // only this thread reads slot threadIdx.x (w = 0 above)
    }
    if (threadIdx.x == 0) *counter = 0u;             // re-armed for the next launch on this stream
    sync();
    return true;
}

// One channel's statistics from the slab totals of slab_reduce<2> / slab_finish<2> (sum (x - shift), sum (x - shift)^2
// in element j = threadIdx.x < 64 of the slab): mean, biased variance, invstd and the running statistics (running_var
// from the unbiased variance), as torch.nn.BatchNorm2d in training mode.
__device__ __forceinline__ void bn_stats_channel(const double* tot, int j, float shift, long long M, float eps,
                                                 float momentum, int c, float* mean_out, float* invstd_out,
                                                 float* running_mean, float* running_var) {
    const int c8 = j >> 3, k = j & 7;
    const double s1 = tot[c8 * 16 + k], s2 = tot[c8 * 16 + 8 + k];
    const double inv_m = 1.0 / (double)M;
    const double md = s1 * inv_m;
    double var = s2 * inv_m - md * md;
    if (var < 0.0) var = 0.0;
    const float mean = (float)((double)shift + md);
    mean_out[c] = mean;
    invstd_out[c] = (float)(1.0 / sqrt(var + (double)eps));
    if (running_mean != nullptr) {
        const double unbiased = M > 1 ? var * ((double)M / (double)(M - 1)) : var;
        running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
        running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unbiased;
    }
}

// One channel's backward sums from the slab totals of slab_reduce<S> / slab_finish<S> (sum g, sum g (x - mean) and,
// S = 3, sum g (x2 - mean2) in element j = threadIdx.x < 64 of the slab): dbeta = sum g, dgamma = invstd * sum
// g (x - mean) in fp64, and with S = 3 the shortcut BN's pair (its dbeta is the same sum).
template <int S>
__device__ __forceinline__ void bn_bwd_channel(const double* tot, int j, int c, const float* invstd, float* dbeta,
                                               float* dgamma, const float* invstd2, float* dbeta2, float* dgamma2) {
    const int c8 = j >> 3, k = j & 7;
    dbeta[c] = (float)tot[c8 * 8 * S + k];
    dgamma[c] = (float)(tot[c8 * 8 * S + 8 + k] * (double)invstd[c]);
    if constexpr (S == 3) {
        dbeta2[c] = (float)tot[c8 * 8 * S + k];
        dgamma2[c] = (float)(tot[c8 * 8 * S + 16 + k] * (double)invstd2[c]);
    }
}

}  // namespace moco
