// Training-mode batch normalisation of channels_last (NHWC) bf16 activations with the ReLU and the residual add of the
// ResNet blocks folded in: the consumer of ShuffleBN's output (ShuffleBN exists so that these batch statistics cannot
// leak the positive pair) and most of the GPU time of a MoCo step when left to ATen's kernels (statistics, transform,
// backward reduce / element-wise, + the separate ReLU and add passes).
//
// Reference call sites: moco/models/resnet.py:42-63 (BasicBlock), :74-102 (Bottleneck: bn -> relu, bn -> relu,
// bn -> += residual -> relu), :114,156-157 (stem), :139-143 (downsample conv -> bn).  Semantics = torch.nn.BatchNorm2d
// in training mode: per-channel mean and BIASED variance over the N*H*W rows, y = (x - mean) * rsqrt(var + eps) * gamma
// + beta, running_mean / running_var updated with `momentum` (running_var from the UNBIASED variance),
// num_batches_tracked += 1; backward = the standard three-term formula.  Everything is computed in fp32 from the bf16
// activations; outputs are rounded to bf16 once.
//
// The activation tensor is a row-major [M, C] matrix (M = N*H*W, C = channels, C * 2 bytes per row).  All four kernels
// are HBM-bound streaming passes:
//   bn_stats_kernel      reads x once        -> mean, invstd (+ running stats)          2 B / element
//   bn_apply_kernel      reads x (+ residual), writes y = relu(x^ * gamma + beta (+ r)) 4 (6) B / element
//   bn_bwd_reduce_kernel reads dy, x (+ y)   -> sum(g), sum(g * x^) = dbeta, dgamma     4 (6) B / element
//   bn_bwd_apply_kernel  reads dy, x (+ y), writes dx (+ d residual)                    6 (10) B / element
// where g = dy masked by the ReLU (the mask is recomputed from x when there is no residual, read from y otherwise).
//
// Reductions: a CTA owns a 64-channel slab (128 contiguous bytes of every row = one 16-byte vector per lane of an
// 8-lane group) and a contiguous range of rows, 32 rows per pass, 4 or 8 passes in flight (see the table of measured
// settings below); per-CTA partials go to a small workspace and the LAST CTA of a slab to finish (ticket counter)
// adds them in a fixed order in fp64 -- deterministic, no atomics on the data.  Sums are taken of (x - x[0, c]) so
// that the variance does not cancel.
// Element-wise passes: thread t keeps the coefficients of its 8 channels in registers (its channel group never
// changes because the grid stride is a multiple of the row length in vectors) and streams 16-byte vectors linearly.
#include "common.cuh"

#include <cuda_bf16.h>

namespace moco {

constexpr int kBnThreads = 256;
constexpr int kBnSlab = 64;                          // channels per reduction CTA
constexpr int kBnLanes = kBnSlab / 8;                // 16-byte vectors per slab row
constexpr int kBnRows = kBnThreads / kBnLanes;       // rows per pass
constexpr int kBnMaxSlabs = 32;                      // C <= 2048
constexpr int kBnMaxPartial = 3 * kBnSlab;           // floats per CTA partial: up to three sums per channel
// (16-byte loads in flight per thread and operand, resident CTAs per SM) of each kernel; every grid is one resident
// wave (tools/bn_kernel_times.py times the variants over the layers of ResNet-50).
constexpr int kBnStatsUnroll = 8, kBnStatsCtas = 2;
constexpr int kBnApplyUnroll = 8, kBnApplyCtas = 2;
constexpr int kBnBwdReduceUnroll = 4, kBnBwdReduceCtas = 2;
constexpr int kBnBwdApplyUnroll = 2, kBnBwdApplyCtas = 3;
constexpr int kBnBwdApplyScUnroll = 2, kBnBwdApplyScCtas = 2;   // with the shortcut BN: 48 coefficients per thread
constexpr int kBnSms = 132;
constexpr int kBnMaxCtas = kBnSms * 4;               // workspace sizing: no reduction grid is larger

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float2 t = __bfloat1622float2(h[k]);
        f[2 * k] = t.x;
        f[2 * k + 1] = t.y;
    }
}

__device__ __forceinline__ uint4 pack8(const float* f) {
    uint4 u;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
    for (int k = 0; k < 4; ++k) h[k] = __floats2bfloat162_rn(f[2 * k], f[2 * k + 1]);
    return u;
}

// Sum the 8 * S per-thread accumulators (S per-channel sums of 8 channels) over the CTA's 32 row groups.  Returns, in
// threads j < 64 * S, element j of the CTA partial: j = v * 8S + k with v = 16-byte lane (8 channels), k < 8 the first
// sum, 8 <= k < 16 the second, 16 <= k < 24 the third.  Each element is added in the same order whatever S is.
template <int S>
__device__ __forceinline__ float slab_reduce(float (&acc)[8 * S], float* red /*[8 * 64S]*/) {
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
    __syncthreads();
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
template <int S>
__device__ __forceinline__ bool slab_finish(float part, float* partial, unsigned int* counter, int slab, int r, int R,
                                            double* tot /*[8 * 64S] shared*/, int* flag /*shared*/) {
    constexpr int P = S * kBnSlab;
    float* mine = partial + ((size_t)slab * R + r) * P;
    if (threadIdx.x < P) mine[threadIdx.x] = part;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int ticket = atomicAdd(counter, 1u);
        *flag = (ticket == (unsigned int)(R - 1));
    }
    __syncthreads();
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
    __syncthreads();
    if (threadIdx.x < P) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < 8; ++w) t += tot[w * P + threadIdx.x];
        __syncwarp();
        tot[threadIdx.x] = t;                        // only this thread reads slot threadIdx.x (w = 0 above)
    }
    if (threadIdx.x == 0) *counter = 0u;             // re-armed for the next launch on this stream
    __syncthreads();
    return true;
}

struct BnStatsArgs {
    const uint4* x;                  // [M, C / 8] vectors
    long long M, passes, ppc;        // ppc = passes per row chunk
    int C, R;
    float eps, momentum;
    float* partial;
    unsigned int* counters;
    float* mean;
    float* invstd;
    float* running_mean;             // nullable
    float* running_var;
    long long* num_batches_tracked;  // nullable
};

template <int kUnroll, int kCtas>
__global__ void __launch_bounds__(kBnThreads, kCtas)
bn_stats_kernel(const BnStatsArgs a) {
    __shared__ float red[8 * 2 * kBnSlab];
    __shared__ double tot[8 * 2 * kBnSlab];
    __shared__ int flag;
    const int slab = blockIdx.x, r = blockIdx.y;
    const int v = threadIdx.x & (kBnLanes - 1), rl = threadIdx.x >> 3;
    const int vec_per_row = a.C >> 3;
    const int colv = slab * kBnLanes + v;
    float sh[8];
    {
        const uint4 u = __ldg(a.x + colv);           // row 0: the shift
        unpack8(u, sh);
    }
    float acc[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) acc[k] = 0.f;
    const long long p0 = (long long)r * a.ppc;
    const long long p1 = (p0 + a.ppc < a.passes) ? p0 + a.ppc : a.passes;
    for (long long p = p0; p < p1; p += kUnroll) {
        uint4 u[kUnroll];
        bool live[kUnroll];
#pragma unroll
        for (int t = 0; t < kUnroll; ++t) {
            const long long row = (p + t) * kBnRows + rl;
            live[t] = (p + t < p1) && row < a.M;
            u[t] = make_uint4(0u, 0u, 0u, 0u);
            if (live[t]) u[t] = __ldg(a.x + row * vec_per_row + colv);
        }
#pragma unroll
        for (int t = 0; t < kUnroll; ++t) {
            if (live[t]) {
                float f[8];
                unpack8(u[t], f);
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const float d = f[k] - sh[k];
                    acc[k] += d;
                    acc[8 + k] = fmaf(d, d, acc[8 + k]);
                }
            }
        }
    }
    const float part = slab_reduce<2>(acc, red);
    if (!slab_finish<2>(part, a.partial, a.counters + slab, slab, r, a.R, tot, &flag)) return;
    if (threadIdx.x < kBnSlab) {
        const int c8 = threadIdx.x >> 3, k = threadIdx.x & 7;
        const int c = slab * kBnSlab + threadIdx.x;
        const double s1 = tot[c8 * 16 + k], s2 = tot[c8 * 16 + 8 + k];
        const double inv_m = 1.0 / (double)a.M;
        const double md = s1 * inv_m;
        double var = s2 * inv_m - md * md;
        if (var < 0.0) var = 0.0;
        const float shift = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(a.x)[c]);
        const float mean = (float)((double)shift + md);
        a.mean[c] = mean;
        a.invstd[c] = (float)(1.0 / sqrt(var + (double)a.eps));
        if (a.running_mean != nullptr) {
            const double unbiased = a.M > 1 ? var * ((double)a.M / (double)(a.M - 1)) : var;
            a.running_mean[c] = (1.f - a.momentum) * a.running_mean[c] + a.momentum * mean;
            a.running_var[c] = (1.f - a.momentum) * a.running_var[c] + a.momentum * (float)unbiased;
        }
    }
    if (slab == 0 && threadIdx.x == 0 && a.num_batches_tracked != nullptr) *a.num_batches_tracked += 1;
}

struct BnApplyArgs {
    const uint4* x;
    const uint4* res;                // nullable; with kShortcut the shortcut convolution's raw output
    uint4* y;
    uint8_t* mask;                   // nullable: bit k of byte j = (y[8j + k] > 0), the ReLU mask of the backward
    long long V;                     // M * C / 8
    int C, relu;
    const float* mean;
    const float* invstd;
    const float* gamma;
    const float* beta;
    const float* mean2;              // kShortcut: the shortcut BN, applied to res and rounded to bf16 before the add
    const float* invstd2;
    const float* gamma2;
    const float* beta2;
};

// 8 mask bits of one vector of y, from the bf16 values as stored (a positive value that rounds to zero is off)
__device__ __forceinline__ unsigned int relu_bits(const uint4& y) {
    float r[8];
    unpack8(y, r);
    unsigned int b = 0u;
#pragma unroll
    for (int k = 0; k < 8; ++k) b |= (r[k] > 0.f ? 1u : 0u) << k;
    return b;
}

template <int kUnroll, int kCtas, bool kShortcut>
__global__ void __launch_bounds__(kBnThreads, kCtas)
bn_apply_kernel(const BnApplyArgs a) {
    const int lanes = a.C >> 3;                      // a power of two <= 256: this thread's channel group is fixed
    const int v = threadIdx.x & (lanes - 1);
    float ca[8], cb[8], ca2[kShortcut ? 8 : 1], cb2[kShortcut ? 8 : 1];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int c = v * 8 + k;
        ca[k] = __ldg(a.gamma + c) * __ldg(a.invstd + c);
        cb[k] = fmaf(-__ldg(a.mean + c), ca[k], __ldg(a.beta + c));
        if constexpr (kShortcut) {
            ca2[k] = __ldg(a.gamma2 + c) * __ldg(a.invstd2 + c);
            cb2[k] = fmaf(-__ldg(a.mean2 + c), ca2[k], __ldg(a.beta2 + c));
        }
    }
    const long long stride = (long long)gridDim.x * kBnThreads;
    const bool has_res = a.res != nullptr;
    for (long long i = (long long)blockIdx.x * kBnThreads + threadIdx.x; i < a.V; i += stride * kUnroll) {
        uint4 u[kUnroll], w[kUnroll];
#pragma unroll
        for (int t = 0; t < kUnroll; ++t) {
            const long long j = i + t * stride;
            u[t] = make_uint4(0u, 0u, 0u, 0u);
            w[t] = make_uint4(0u, 0u, 0u, 0u);
            if (j < a.V) {
                u[t] = __ldg(a.x + j);
                if (has_res) w[t] = __ldg(a.res + j);
            }
        }
#pragma unroll
        for (int t = 0; t < kUnroll; ++t) {
            const long long j = i + t * stride;
            if (j < a.V) {
                float f[8], g[8];
                unpack8(u[t], f);
                unpack8(w[t], g);
                if constexpr (kShortcut) {
                    // what the shortcut BN's own pass stores (its "+ residual" is +0.f) and the add reads back
#pragma unroll
                    for (int k = 0; k < 8; ++k)
                        g[k] = __bfloat162float(__float2bfloat16_rn(__fadd_rn(fmaf(g[k], ca2[k], cb2[k]), 0.f)));
                }
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    float z = fmaf(f[k], ca[k], cb[k]) + g[k];
                    if (a.relu) z = fmaxf(z, 0.f);
                    f[k] = z;
                }
                const uint4 out = pack8(f);
                a.y[j] = out;
                if (a.mask != nullptr) a.mask[j] = (uint8_t)relu_bits(out);
            }
        }
    }
}

// how the ReLU mask of the backward is obtained
enum { kMaskNone = 0, kMaskFromY = 1, kMaskFromX = 2, kMaskFromBits = 3 };

struct BnBwdReduceArgs {
    const uint4* dy;
    const uint4* x;
    const uint4* y;                  // kMaskFromY only
    const uint8_t* mbits;            // kMaskFromBits only: the forward's mask bytes
    const uint4* x2;                 // kShortcut: the shortcut BN's input
    long long M, passes, ppc;
    int C, R, mask;
    float* partial;
    unsigned int* counters;
    const float* mean;
    const float* invstd;
    const float* gamma;
    const float* beta;
    const float* mean2;              // kShortcut
    const float* invstd2;
    float* sum_dy;                   // = dbeta
    float* sum_dy_xhat;              // = dgamma
    float* sum_dy2;                  // kShortcut: = the shortcut BN's dbeta (the same sum)
    float* sum_dy_xhat2;             // kShortcut: = the shortcut BN's dgamma
};

__device__ __forceinline__ bool mask_on(int mode, float y, unsigned int bits, int k, float x, float ca, float cb) {
    if (mode == kMaskFromY) return y > 0.f;
    if (mode == kMaskFromX) return fmaf(x, ca, cb) > 0.f;
    if (mode == kMaskFromBits) return (bits >> k) & 1u;
    return true;
}

// kShortcut: the block's bn3 and the shortcut BN of a downsample block, both fed by the same masked gradient g: a
// third sum, g * (x2 - mean2), taken in the same row / slab plan and per-thread order as the shortcut's own reduction.
template <int kUnroll, int kCtas, bool kShortcut>
__global__ void __launch_bounds__(kBnThreads, kCtas)
bn_bwd_reduce_kernel(const BnBwdReduceArgs a) {
    constexpr int S = kShortcut ? 3 : 2;
    __shared__ float red[8 * S * kBnSlab];
    __shared__ double tot[8 * S * kBnSlab];
    __shared__ int flag;
    const int slab = blockIdx.x, r = blockIdx.y;
    const int v = threadIdx.x & (kBnLanes - 1), rl = threadIdx.x >> 3;
    const int vec_per_row = a.C >> 3;
    const int colv = slab * kBnLanes + v;
    const int mode = kShortcut ? (int)kMaskFromBits : a.mask;      // a downsample block's bn3 always has its mask bits
    float mu[8], ca[8], cb[8], mu2[kShortcut ? 8 : 1]; // sum(g x^) = invstd * sum(g (x - mean)): invstd applied at the end
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int c = colv * 8 + k;
        mu[k] = __ldg(a.mean + c);
        ca[k] = cb[k] = 0.f;
        if (mode == kMaskFromX) {
            ca[k] = __ldg(a.gamma + c) * __ldg(a.invstd + c);
            cb[k] = fmaf(-mu[k], ca[k], __ldg(a.beta + c));
        }
        if constexpr (kShortcut) mu2[k] = __ldg(a.mean2 + c);
    }
    float acc[8 * S];
#pragma unroll
    for (int k = 0; k < 8 * S; ++k) acc[k] = 0.f;
    const long long p0 = (long long)r * a.ppc;
    const long long p1 = (p0 + a.ppc < a.passes) ? p0 + a.ppc : a.passes;
    for (long long p = p0; p < p1; p += kUnroll) {
        uint4 ud[kUnroll], ux[kUnroll], uy[kUnroll], u2[kShortcut ? kUnroll : 1];
        unsigned int mb[kUnroll];
        bool live[kUnroll];
#pragma unroll
        for (int t = 0; t < kUnroll; ++t) {
            const long long row = (p + t) * kBnRows + rl;
            live[t] = (p + t < p1) && row < a.M;
            ud[t] = ux[t] = uy[t] = make_uint4(0u, 0u, 0u, 0u);
            if constexpr (kShortcut) u2[t] = make_uint4(0u, 0u, 0u, 0u);
            mb[t] = 0u;
            if (live[t]) {
                const long long j = row * vec_per_row + colv;
                ud[t] = __ldg(a.dy + j);
                ux[t] = __ldg(a.x + j);
                if (mode == kMaskFromY) uy[t] = __ldg(a.y + j);
                if (mode == kMaskFromBits) mb[t] = __ldg(a.mbits + j);
                if constexpr (kShortcut) u2[t] = __ldg(a.x2 + j);
            }
        }
#pragma unroll
        for (int t = 0; t < kUnroll; ++t) {
            if (live[t]) {
                float d[8], f[8], yy[8], f2[kShortcut ? 8 : 1];
                unpack8(ud[t], d);
                unpack8(ux[t], f);
                unpack8(uy[t], yy);
                if constexpr (kShortcut) unpack8(u2[t], f2);
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const float g = mask_on(mode, yy[k], mb[t], k, f[k], ca[k], cb[k]) ? d[k] : 0.f;
                    acc[k] += g;
                    acc[8 + k] = fmaf(g, f[k] - mu[k], acc[8 + k]);
                    if constexpr (kShortcut) acc[16 + k] = fmaf(g, f2[k] - mu2[k], acc[16 + k]);
                }
            }
        }
    }
    const float part = slab_reduce<S>(acc, red);
    if (!slab_finish<S>(part, a.partial, a.counters + slab, slab, r, a.R, tot, &flag)) return;
    if (threadIdx.x < kBnSlab) {
        const int c8 = threadIdx.x >> 3, k = threadIdx.x & 7;
        const int c = slab * kBnSlab + threadIdx.x;
        a.sum_dy[c] = (float)tot[c8 * 8 * S + k];
        a.sum_dy_xhat[c] = (float)(tot[c8 * 8 * S + 8 + k] * (double)a.invstd[c]);
        if constexpr (kShortcut) {
            a.sum_dy2[c] = (float)tot[c8 * 8 * S + k];
            a.sum_dy_xhat2[c] = (float)(tot[c8 * 8 * S + 16 + k] * (double)a.invstd2[c]);
        }
    }
}

struct BnBwdApplyArgs {
    const uint4* dy;
    const uint4* x;
    const uint4* y;                  // kMaskFromY only
    const uint8_t* mbits;            // kMaskFromBits only
    const uint4* x2;                 // kShortcut: the shortcut BN's input
    uint4* dx;
    uint4* dres;                     // nullable: the masked gradient, for the residual branch
    uint4* dx2;                      // kShortcut: the shortcut BN's input gradient
    long long V;
    int C, mask;
    float inv_m;
    const float* mean;
    const float* invstd;
    const float* gamma;
    const float* beta;
    const float* sum_dy;
    const float* sum_dy_xhat;
    const float* mean2;              // kShortcut
    const float* invstd2;
    const float* gamma2;
    const float* sum_dy_xhat2;
};

// dx = k1 * (g - m1 - x^ * m2),  k1 = gamma * invstd, m1 = sum(g) / M, m2 = sum(g x^) / M, x^ = (x - mean) * invstd
//    = cA * g + cB * x + cD
__device__ __forceinline__ void bwd_coefs(float gamma, float mu, float is, float sum_dy, float sum_dy_xhat, float inv_m,
                                          float& cA, float& cB, float& cD) {
    const float k1 = gamma * is;
    const float m1 = sum_dy * inv_m, m2 = sum_dy_xhat * inv_m;
    cA = k1;
    cB = -k1 * m2 * is;
    cD = fmaf(-cB, mu, -k1 * m1);
}

template <int kUnroll, int kCtas, bool kShortcut>
__global__ void __launch_bounds__(kBnThreads, kCtas)
bn_bwd_apply_kernel(const BnBwdApplyArgs a) {
    const int lanes = a.C >> 3;
    const int v = threadIdx.x & (lanes - 1);
    const int mode = kShortcut ? (int)kMaskFromBits : a.mask;
    constexpr int K2 = kShortcut ? 8 : 1;
    float cA[8], cB[8], cD[8], ca[8], cb[8], cA2[K2], cB2[K2], cD2[K2];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int c = v * 8 + k;
        const float mu = __ldg(a.mean + c), is = __ldg(a.invstd + c);
        bwd_coefs(__ldg(a.gamma + c), mu, is, __ldg(a.sum_dy + c), __ldg(a.sum_dy_xhat + c), a.inv_m, cA[k], cB[k], cD[k]);
        ca[k] = cA[k];
        cb[k] = mode == kMaskFromX ? fmaf(-mu, cA[k], __ldg(a.beta + c)) : 0.f;
        if constexpr (kShortcut)
            bwd_coefs(__ldg(a.gamma2 + c), __ldg(a.mean2 + c), __ldg(a.invstd2 + c), __ldg(a.sum_dy + c),
                      __ldg(a.sum_dy_xhat2 + c), a.inv_m, cA2[k], cB2[k], cD2[k]);
    }
    const long long stride = (long long)gridDim.x * kBnThreads;
    for (long long i = (long long)blockIdx.x * kBnThreads + threadIdx.x; i < a.V; i += stride * kUnroll) {
        uint4 ud[kUnroll], ux[kUnroll], uy[kUnroll], u2[kShortcut ? kUnroll : 1];
        unsigned int mb[kUnroll];
#pragma unroll
        for (int t = 0; t < kUnroll; ++t) {
            const long long j = i + t * stride;
            ud[t] = ux[t] = uy[t] = make_uint4(0u, 0u, 0u, 0u);
            if constexpr (kShortcut) u2[t] = make_uint4(0u, 0u, 0u, 0u);
            mb[t] = 0u;
            if (j < a.V) {
                ud[t] = __ldg(a.dy + j);
                ux[t] = __ldg(a.x + j);
                if (mode == kMaskFromY) uy[t] = __ldg(a.y + j);
                if (mode == kMaskFromBits) mb[t] = __ldg(a.mbits + j);
                if constexpr (kShortcut) u2[t] = __ldg(a.x2 + j);
            }
        }
#pragma unroll
        for (int t = 0; t < kUnroll; ++t) {
            const long long j = i + t * stride;
            if (j < a.V) {
                float d[8], f[8], yy[8], o[8];
                unpack8(ud[t], d);
                unpack8(ux[t], f);
                unpack8(uy[t], yy);
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const float g = mask_on(mode, yy[k], mb[t], k, f[k], ca[k], cb[k]) ? d[k] : 0.f;
                    d[k] = g;
                    o[k] = fmaf(cA[k], g, fmaf(cB[k], f[k], cD[k]));
                }
                a.dx[j] = pack8(o);
                if constexpr (kShortcut) {
                    unpack8(u2[t], f);
#pragma unroll
                    for (int k = 0; k < 8; ++k) o[k] = fmaf(cA2[k], d[k], fmaf(cB2[k], f[k], cD2[k]));
                    a.dx2[j] = pack8(o);
                } else if (a.dres != nullptr) {
                    a.dres[j] = pack8(d);
                }
            }
        }
    }
}

// ---- frozen (eval-mode) BatchNorm -----------------------------------------------------------------------------------
// The per-channel scale / shift are folded by the caller from the running statistics; there is no statistics pass and
// no backward.  Arithmetic is the header's numerical contract: no FMA contraction, so that separate fp32 torch ops
// reproduce every bit.

struct BnEvalArgs {
    const uint4* x;
    const uint4* res;                // nullable; with kShortcut the shortcut convolution's raw output
    uint4* y;                        // element-wise pass
    float* feat;                     // pooled pass: fp32 [N, C]
    long long V;                     // element-wise: M * C / 8 vectors; pooled: N * C / 8 (one (image, vector) each)
    int C, HW, relu;
    const float* scale;
    const float* shift;
    const float* scale2;             // kShortcut
    const float* shift2;
};

// z = relu?((x * s + t) [+ r]) in fp32, r = bf16((res * s2 + t2)) with a shortcut BN; returned unrounded
template <bool kShortcut>
__device__ __forceinline__ void bn_eval8(const uint4& ux, const uint4& ur, bool has_res, int relu, const float* s,
                                         const float* t, const float* s2, const float* t2, float* z) {
    float f[8], g[8];
    unpack8(ux, f);
    unpack8(ur, g);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        float v = __fadd_rn(__fmul_rn(f[k], s[k]), t[k]);
        if (has_res) {
            float r = g[k];
            if constexpr (kShortcut) r = __bfloat162float(__float2bfloat16_rn(__fadd_rn(__fmul_rn(r, s2[k]), t2[k])));
            v = __fadd_rn(v, r);
        }
        if (relu) v = v > 0.f ? v : 0.f;
        z[k] = v;
    }
}

template <bool kShortcut>
__device__ __forceinline__ void bn_eval_coefs(const BnEvalArgs& a, int v, float* s, float* t, float* s2, float* t2) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int c = v * 8 + k;
        s[k] = __ldg(a.scale + c);
        t[k] = __ldg(a.shift + c);
        if constexpr (kShortcut) { s2[k] = __ldg(a.scale2 + c); t2[k] = __ldg(a.shift2 + c); }
    }
}

template <bool kShortcut>
__global__ void __launch_bounds__(kBnThreads, kBnApplyCtas)
bn_eval_kernel(const BnEvalArgs a) {
    const int v = threadIdx.x & ((a.C >> 3) - 1);    // fixed channel group, as in bn_apply_kernel
    float s[8], t[8], s2[kShortcut ? 8 : 1], t2[kShortcut ? 8 : 1];
    bn_eval_coefs<kShortcut>(a, v, s, t, s2, t2);
    const long long stride = (long long)gridDim.x * kBnThreads;
    const bool has_res = a.res != nullptr;
    for (long long i = (long long)blockIdx.x * kBnThreads + threadIdx.x; i < a.V; i += stride * kBnApplyUnroll) {
        uint4 u[kBnApplyUnroll], w[kBnApplyUnroll];
#pragma unroll
        for (int k = 0; k < kBnApplyUnroll; ++k) {
            const long long j = i + k * stride;
            u[k] = w[k] = make_uint4(0u, 0u, 0u, 0u);
            if (j < a.V) {
                u[k] = __ldg(a.x + j);
                if (has_res) w[k] = __ldg(a.res + j);
            }
        }
#pragma unroll
        for (int k = 0; k < kBnApplyUnroll; ++k) {
            const long long j = i + k * stride;
            if (j < a.V) {
                float z[8];
                bn_eval8<kShortcut>(u[k], w[k], has_res, a.relu, s, t, s2, t2, z);
                a.y[j] = pack8(z);
            }
        }
    }
}

// The last block's BatchNorm (+ add + ReLU) followed by the global average pool: thread (n, v) walks the HW pixels of
// image n in increasing order, adds the bf16-rounded outputs in fp32 and divides once.  The map is never written.
// The pixel order is the contract, so the parallelism is N * C / 8 threads; 64-thread CTAs spread a small batch over
// the SMs (N = 32 at C = 2048: 128 CTAs rather than 32 of 256 threads).
constexpr int kBnPoolUnroll = 7;
constexpr int kBnPoolThreads = 64;

template <bool kShortcut>
__global__ void __launch_bounds__(kBnPoolThreads, 8)   // 512 threads per SM: N = 256, C = 2048 is one wave
bn_eval_avgpool_kernel(const BnEvalArgs a) {
    const long long o = (long long)blockIdx.x * kBnPoolThreads + threadIdx.x;
    if (o >= a.V) return;
    const int lanes = a.C >> 3;
    const int v = (int)(o & (lanes - 1));
    const long long n = o / lanes;
    float s[8], t[8], s2[kShortcut ? 8 : 1], t2[kShortcut ? 8 : 1];
    bn_eval_coefs<kShortcut>(a, v, s, t, s2, t2);
    const bool has_res = a.res != nullptr;
    const long long base = n * a.HW * lanes + v;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    for (int p0 = 0; p0 < a.HW; p0 += kBnPoolUnroll) {
        uint4 u[kBnPoolUnroll], w[kBnPoolUnroll];
#pragma unroll
        for (int q = 0; q < kBnPoolUnroll; ++q) {
            u[q] = w[q] = make_uint4(0u, 0u, 0u, 0u);
            if (p0 + q < a.HW) {
                const long long j = base + (long long)(p0 + q) * lanes;
                u[q] = __ldg(a.x + j);
                if (has_res) w[q] = __ldg(a.res + j);
            }
        }
#pragma unroll
        for (int q = 0; q < kBnPoolUnroll; ++q) {
            if (p0 + q < a.HW) {
                float z[8];
                bn_eval8<kShortcut>(u[q], w[q], has_res, a.relu, s, t, s2, t2, z);
#pragma unroll
                for (int k = 0; k < 8; ++k) acc[k] = __fadd_rn(acc[k], __bfloat162float(__float2bfloat16_rn(z[k])));
            }
        }
    }
    const float hw = (float)a.HW;
    float4* out = reinterpret_cast<float4*>(a.feat + n * a.C + v * 8);
    out[0] = make_float4(__fdiv_rn(acc[0], hw), __fdiv_rn(acc[1], hw), __fdiv_rn(acc[2], hw), __fdiv_rn(acc[3], hw));
    out[1] = make_float4(__fdiv_rn(acc[4], hw), __fdiv_rn(acc[5], hw), __fdiv_rn(acc[6], hw), __fdiv_rn(acc[7], hw));
}

// ---- host side ------------------------------------------------------------------------------------------------------

size_t bn_workspace_bytes() { return 256 + (size_t)kBnMaxCtas * kBnMaxPartial * sizeof(float); }

static bool bn_shape_ok(long long M, int C) {
    if (M < 1 || C < kBnSlab || C > kBnSlab * kBnMaxSlabs) return false;
    return (C & (C - 1)) == 0;                       // 64 .. 2048, a power of two (256 % (C / 8) == 0)
}

static void bn_reduce_plan(long long M, int C, int unroll, int ctas_per_sm, long long* passes, long long* ppc, int* R) {
    const int slabs = C / kBnSlab;
    const long long np = (M + kBnRows - 1) / kBnRows;
    long long r = kBnSms * ctas_per_sm / slabs;
    const long long want = (np + unroll - 1) / unroll;            // at least one unrolled trip per CTA
    if (r > want) r = want;
    if (r < 1) r = 1;
    long long per = (np + r - 1) / r;
    per = (per + unroll - 1) / unroll * unroll;
    r = (np + per - 1) / per;
    *passes = np; *ppc = per; *R = (int)r;
}

static int bn_apply_grid(long long V, int unroll, int ctas_per_sm) {
    long long g = (V + (long long)kBnThreads * unroll - 1) / ((long long)kBnThreads * unroll);
    if (g > kBnSms * ctas_per_sm) g = kBnSms * ctas_per_sm;
    if (g < 1) g = 1;
    return (int)g;
}

template <int U, int CT>
static cudaError_t run_stats(BnStatsArgs& s, cudaStream_t stream) {
    bn_reduce_plan(s.M, s.C, U, CT, &s.passes, &s.ppc, &s.R);
    bn_stats_kernel<U, CT><<<dim3(s.C / kBnSlab, s.R), kBnThreads, 0, stream>>>(s);
    return cudaGetLastError();
}
template <int U, int CT, bool SC>
static cudaError_t run_apply(BnApplyArgs& p, cudaStream_t stream) {
    bn_apply_kernel<U, CT, SC><<<bn_apply_grid(p.V, U, CT), kBnThreads, 0, stream>>>(p);
    return cudaGetLastError();
}
template <int U, int CT, bool SC>
static cudaError_t run_bwd_reduce(BnBwdReduceArgs& s, cudaStream_t stream) {
    bn_reduce_plan(s.M, s.C, U, CT, &s.passes, &s.ppc, &s.R);
    bn_bwd_reduce_kernel<U, CT, SC><<<dim3(s.C / kBnSlab, s.R), kBnThreads, 0, stream>>>(s);
    return cudaGetLastError();
}
template <int U, int CT, bool SC>
static cudaError_t run_bwd_apply(BnBwdApplyArgs& p, cudaStream_t stream) {
    bn_bwd_apply_kernel<U, CT, SC><<<bn_apply_grid(p.V, U, CT), kBnThreads, 0, stream>>>(p);
    return cudaGetLastError();
}

static cudaError_t stats_pass(const void* x, long long M, int C, float* running_mean, float* running_var, long long* nbt,
                              float momentum, float eps, float* save_mean, float* save_invstd, void* ws,
                              cudaStream_t stream) {
    BnStatsArgs s{};
    s.x = static_cast<const uint4*>(x);
    s.M = M; s.C = C;
    s.eps = eps; s.momentum = momentum;
    s.counters = static_cast<unsigned int*>(ws);
    s.partial = reinterpret_cast<float*>(static_cast<uint8_t*>(ws) + 256);
    s.mean = save_mean; s.invstd = save_invstd;
    s.running_mean = running_mean; s.running_var = running_var; s.num_batches_tracked = nbt;
    return run_stats<kBnStatsUnroll, kBnStatsCtas>(s, stream);
}

cudaError_t launch_bn_fwd_train(const void* x, const void* res, void* y, long long M, int C, const float* gamma,
                                const float* beta, float* running_mean, float* running_var, long long* nbt, float momentum,
                                float eps, int relu, float* save_mean, float* save_invstd, void* ws, cudaStream_t stream) {
    if (!bn_shape_ok(M, C)) return cudaErrorNotSupported;
    cudaError_t e = stats_pass(x, M, C, running_mean, running_var, nbt, momentum, eps, save_mean, save_invstd, ws, stream);
    if (e != cudaSuccess) return e;
    BnApplyArgs p{};
    p.x = static_cast<const uint4*>(x); p.res = static_cast<const uint4*>(res); p.y = static_cast<uint4*>(y);
    p.V = M * (C >> 3); p.C = C; p.relu = relu;
    p.mean = save_mean; p.invstd = save_invstd; p.gamma = gamma; p.beta = beta;
    return run_apply<kBnApplyUnroll, kBnApplyCtas, false>(p, stream);
}

cudaError_t launch_bn_bwd(const void* dy, const void* x, const void* y, long long M, int C, const float* gamma,
                          const float* beta, const float* save_mean, const float* save_invstd, int relu, int has_residual,
                          void* dx, void* dres, float* dgamma, float* dbeta, void* ws, cudaStream_t stream) {
    if (!bn_shape_ok(M, C)) return cudaErrorNotSupported;
    const int mask = !relu ? kMaskNone : (has_residual ? kMaskFromY : kMaskFromX);
    if (mask == kMaskFromY && y == nullptr) return cudaErrorInvalidValue;
    BnBwdReduceArgs s{};
    s.dy = static_cast<const uint4*>(dy); s.x = static_cast<const uint4*>(x); s.y = static_cast<const uint4*>(y);
    s.M = M; s.C = C; s.mask = mask;
    s.counters = static_cast<unsigned int*>(ws);
    s.partial = reinterpret_cast<float*>(static_cast<uint8_t*>(ws) + 256);
    s.mean = save_mean; s.invstd = save_invstd; s.gamma = gamma; s.beta = beta;
    s.sum_dy = dbeta; s.sum_dy_xhat = dgamma;
    cudaError_t e = run_bwd_reduce<kBnBwdReduceUnroll, kBnBwdReduceCtas, false>(s, stream);
    if (e != cudaSuccess) return e;
    BnBwdApplyArgs p{};
    p.dy = s.dy; p.x = s.x; p.y = s.y; p.dx = static_cast<uint4*>(dx); p.dres = static_cast<uint4*>(dres);
    p.V = M * (C >> 3); p.C = C; p.mask = mask; p.inv_m = (float)(1.0 / (double)M);
    p.mean = save_mean; p.invstd = save_invstd; p.gamma = gamma; p.beta = beta;
    p.sum_dy = dbeta; p.sum_dy_xhat = dgamma;
    return run_bwd_apply<kBnBwdApplyUnroll, kBnBwdApplyCtas, false>(p, stream);
}

cudaError_t launch_bn_add_relu_fwd(const void* x, const void* res, void* y, void* mask, long long M, int C,
                                   const BnLayer& bn, const BnLayer* sc, void* ws, cudaStream_t stream) {
    if (!bn_shape_ok(M, C)) return cudaErrorNotSupported;
    cudaError_t e = stats_pass(x, M, C, bn.running_mean, bn.running_var, bn.num_batches_tracked, bn.momentum, bn.eps,
                               bn.save_mean, bn.save_invstd, ws, stream);
    if (e == cudaSuccess && sc != nullptr)
        e = stats_pass(res, M, C, sc->running_mean, sc->running_var, sc->num_batches_tracked, sc->momentum, sc->eps,
                       sc->save_mean, sc->save_invstd, ws, stream);
    if (e != cudaSuccess) return e;
    BnApplyArgs p{};
    p.x = static_cast<const uint4*>(x); p.res = static_cast<const uint4*>(res); p.y = static_cast<uint4*>(y);
    p.mask = static_cast<uint8_t*>(mask);
    p.V = M * (C >> 3); p.C = C; p.relu = 1;
    p.mean = bn.save_mean; p.invstd = bn.save_invstd; p.gamma = bn.gamma; p.beta = bn.beta;
    if (sc == nullptr) return run_apply<kBnApplyUnroll, kBnApplyCtas, false>(p, stream);
    p.mean2 = sc->save_mean; p.invstd2 = sc->save_invstd; p.gamma2 = sc->gamma; p.beta2 = sc->beta;
    return run_apply<kBnApplyUnroll, kBnApplyCtas, true>(p, stream);
}

cudaError_t launch_bn_add_relu_bwd(const void* dy, const void* x, const void* res, const void* mask, long long M, int C,
                                   const BnLayer& bn, const BnLayer* sc, void* dx, void* dres, void* ws,
                                   cudaStream_t stream) {
    if (!bn_shape_ok(M, C)) return cudaErrorNotSupported;
    BnBwdReduceArgs s{};
    s.dy = static_cast<const uint4*>(dy); s.x = static_cast<const uint4*>(x);
    s.mbits = static_cast<const uint8_t*>(mask);
    s.M = M; s.C = C; s.mask = kMaskFromBits;
    s.counters = static_cast<unsigned int*>(ws);
    s.partial = reinterpret_cast<float*>(static_cast<uint8_t*>(ws) + 256);
    s.mean = bn.save_mean; s.invstd = bn.save_invstd; s.gamma = bn.gamma;
    s.sum_dy = bn.dbeta; s.sum_dy_xhat = bn.dgamma;
    BnBwdApplyArgs p{};
    p.dy = s.dy; p.x = s.x; p.mbits = s.mbits; p.dx = static_cast<uint4*>(dx);
    p.V = M * (C >> 3); p.C = C; p.mask = kMaskFromBits; p.inv_m = (float)(1.0 / (double)M);
    p.mean = bn.save_mean; p.invstd = bn.save_invstd; p.gamma = bn.gamma;
    p.sum_dy = bn.dbeta; p.sum_dy_xhat = bn.dgamma;
    cudaError_t e;
    if (sc == nullptr) {
        p.dres = static_cast<uint4*>(dres);
        e = run_bwd_reduce<kBnBwdReduceUnroll, kBnBwdReduceCtas, false>(s, stream);
        if (e != cudaSuccess) return e;
        return run_bwd_apply<kBnBwdApplyUnroll, kBnBwdApplyCtas, false>(p, stream);
    }
    s.x2 = static_cast<const uint4*>(res);
    s.mean2 = sc->save_mean; s.invstd2 = sc->save_invstd;
    s.sum_dy2 = sc->dbeta; s.sum_dy_xhat2 = sc->dgamma;
    e = run_bwd_reduce<kBnBwdReduceUnroll, kBnBwdReduceCtas, true>(s, stream);
    if (e != cudaSuccess) return e;
    p.x2 = s.x2; p.dx2 = static_cast<uint4*>(dres);
    p.mean2 = sc->save_mean; p.invstd2 = sc->save_invstd; p.gamma2 = sc->gamma; p.sum_dy_xhat2 = sc->dgamma;
    return run_bwd_apply<kBnBwdApplyScUnroll, kBnBwdApplyScCtas, true>(p, stream);
}

cudaError_t launch_bn_relu_maxpool_fwd(const void* x, void* y, void* taps, int N, int H, int W, int C, const BnLayer& bn,
                                       void* ws, cudaStream_t stream) {
    const long long M = (long long)N * H * W;
    if (N < 1 || H < 1 || W < 1 || !bn_shape_ok(M, C)) return cudaErrorNotSupported;
    cudaError_t e = stats_pass(x, M, C, bn.running_mean, bn.running_var, bn.num_batches_tracked, bn.momentum, bn.eps,
                               bn.save_mean, bn.save_invstd, ws, stream);
    if (e != cudaSuccess) return e;
    return launch_maxpool_fwd(x, y, taps, N, H, W, C, stream, bn.save_mean, bn.save_invstd, bn.gamma, bn.beta);
}

static BnEvalArgs eval_args(const void* x, const void* res, int C, const float* scale, const float* shift, int relu,
                            const float* sc_scale, const float* sc_shift) {
    BnEvalArgs a{};
    a.x = static_cast<const uint4*>(x); a.res = static_cast<const uint4*>(res);
    a.C = C; a.relu = relu;
    a.scale = scale; a.shift = shift; a.scale2 = sc_scale; a.shift2 = sc_shift;
    return a;
}

cudaError_t launch_bn_eval_act(const void* x, const void* res, void* y, long long M, int C, const float* scale,
                               const float* shift, int relu, const float* sc_scale, const float* sc_shift,
                               cudaStream_t stream) {
    if (!bn_shape_ok(M, C)) return cudaErrorNotSupported;
    BnEvalArgs a = eval_args(x, res, C, scale, shift, relu, sc_scale, sc_shift);
    a.y = static_cast<uint4*>(y);
    a.V = M * (C >> 3);
    const int grid = bn_apply_grid(a.V, kBnApplyUnroll, kBnApplyCtas);
    if (sc_scale != nullptr) bn_eval_kernel<true><<<grid, kBnThreads, 0, stream>>>(a);
    else bn_eval_kernel<false><<<grid, kBnThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_bn_eval_act_avgpool(const void* x, const void* res, float* feat, int N, int HW, int C,
                                       const float* scale, const float* shift, int relu, const float* sc_scale,
                                       const float* sc_shift, cudaStream_t stream) {
    if (N < 1 || HW < 1 || !bn_shape_ok((long long)N * HW, C)) return cudaErrorNotSupported;
    BnEvalArgs a = eval_args(x, res, C, scale, shift, relu, sc_scale, sc_shift);
    a.feat = feat;
    a.HW = HW;
    a.V = (long long)N * (C >> 3);
    const long long blocks = (a.V + kBnPoolThreads - 1) / kBnPoolThreads;
    if (blocks > 0x7fffffffLL) return cudaErrorNotSupported;
    if (sc_scale != nullptr) bn_eval_avgpool_kernel<true><<<(unsigned int)blocks, kBnPoolThreads, 0, stream>>>(a);
    else bn_eval_avgpool_kernel<false><<<(unsigned int)blocks, kBnPoolThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_bn_relu_maxpool_eval(const void* x, void* y, int N, int H, int W, int C, const float* scale,
                                        const float* shift, cudaStream_t stream) {
    if (N < 1 || H < 1 || W < 1 || !bn_shape_ok((long long)N * H * W, C)) return cudaErrorNotSupported;
    return launch_maxpool_fwd(x, y, nullptr, N, H, W, C, stream, nullptr, nullptr, nullptr, nullptr, scale, shift);
}

}  // namespace moco
