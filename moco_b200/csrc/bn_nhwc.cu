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
// where g = dy masked by the ReLU (the mask is recomputed from x when there is no residual -- y > 0 of the bf16 value
// the forward stores -- and read from y otherwise).
// A block output's gradient may arrive in two parts (the next block's first convolution and its residual branch):
// both backward passes then read dy and dy2 and use bf16(dy + dy2), +2 B / element each (kSum, moco_bn_add_relu_bwd2).
//
// Reductions: a CTA owns a 64-channel slab (128 contiguous bytes of every row = one 16-byte vector per lane of an
// 8-lane group) and a contiguous range of rows, 32 rows per pass, 4 or 8 passes in flight (see the table of measured
// settings below); per-CTA partials go to a small workspace and the LAST CTA of a slab to finish (ticket counter)
// adds them in a fixed order in fp64 -- deterministic, no atomics on the data.  Sums are taken of (x - x[0, c]) so
// that the variance does not cancel.
// Element-wise passes: thread t keeps the coefficients of its 8 channels in registers (its channel group never
// changes because the grid stride is a multiple of the row length in vectors) and streams 16-byte vectors linearly.
#include "bn_reduce.cuh"
#include "common.cuh"

#include <cuda_bf16.h>

namespace moco {

constexpr int kBnMaxSlabs = 32;                      // C <= 2048
constexpr int kBnMaxPartial = 3 * kBnSlab;           // floats per CTA partial: up to three sums per channel
// (16-byte loads in flight per thread and operand, resident CTAs per SM) of each kernel; every grid is one resident
// wave (tools/bn_kernel_times.py times the variants over the layers of ResNet-50).
constexpr int kBnApplyUnroll = 8, kBnApplyCtas = 2;
constexpr int kBnBwdApplyUnroll = 2, kBnBwdApplyCtas = 3;
constexpr int kBnBwdApplyScUnroll = 2, kBnBwdApplyScCtas = 2;   // with the shortcut BN: 48 coefficients per thread
constexpr int kBnBwdApplySumUnroll = 2, kBnBwdApplySumCtas = 2; // with a second gradient (dy2): spills at 3 CTAs / SM
constexpr int kBnSms = 132;
constexpr int kBnMaxCtas = kBnSms * 4;               // workspace sizing: no reduction grid is larger

__device__ __forceinline__ uint4 pack8(const float* f) {
    uint4 u;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
    for (int k = 0; k < 4; ++k) h[k] = __floats2bfloat162_rn(f[2 * k], f[2 * k + 1]);
    return u;
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
        const int c = slab * kBnSlab + threadIdx.x;
        bn_stats_channel(tot, threadIdx.x, __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(a.x)[c]), a.M, a.eps,
                         a.momentum, c, a.mean, a.invstd, a.running_mean, a.running_var);
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

// kSum: the incoming gradient is the sum of two, dy + dy2, rounded to bf16 once before any other use -- what autograd's
// bf16 add of the two branch gradients of a block's input would have stored (fp32 add, one rounding); never written
__device__ __forceinline__ void sum_grads(float* d, const uint4& u2) {
    float d2[8];
    unpack8(u2, d2);
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] = __bfloat162float(__float2bfloat16_rn(__fadd_rn(d[k], d2[k])));
}

struct BnBwdReduceArgs {
    const uint4* dy;
    const uint4* dy2;                // kSum only: the second gradient of y
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

// kMaskFromX: y > 0 of the bf16 value bn_apply_kernel stores (relu_bits' rule), so a positive pre-activation that
// rounds to zero is off.  bf16 rounds z to zero iff z <= 2^-134, half its smallest subnormal (the tie goes to the even
// zero); the comparison with that constant needs no register for the rounded value (one more spills the
// 3-CTA / SM apply kernel).
__device__ __forceinline__ bool mask_on(int mode, float y, unsigned int bits, int k, float x, float ca, float cb) {
    if (mode == kMaskFromY) return y > 0.f;
    if (mode == kMaskFromX) return fmaf(x, ca, cb) > 0x1p-134f;
    if (mode == kMaskFromBits) return (bits >> k) & 1u;
    return true;
}

// kShortcut: the block's bn3 and the shortcut BN of a downsample block, both fed by the same masked gradient g: a
// third sum, g * (x2 - mean2), taken in the same row / slab plan and per-thread order as the shortcut's own reduction.
template <int kUnroll, int kCtas, bool kShortcut, bool kSum>
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
        uint4 ud[kUnroll], ux[kUnroll], uy[kUnroll], u2[kShortcut ? kUnroll : 1], us[kSum ? kUnroll : 1];
        unsigned int mb[kUnroll];
        bool live[kUnroll];
#pragma unroll
        for (int t = 0; t < kUnroll; ++t) {
            const long long row = (p + t) * kBnRows + rl;
            live[t] = (p + t < p1) && row < a.M;
            ud[t] = ux[t] = uy[t] = make_uint4(0u, 0u, 0u, 0u);
            if constexpr (kShortcut) u2[t] = make_uint4(0u, 0u, 0u, 0u);
            if constexpr (kSum) us[t] = make_uint4(0u, 0u, 0u, 0u);
            mb[t] = 0u;
            if (live[t]) {
                const long long j = row * vec_per_row + colv;
                ud[t] = __ldg(a.dy + j);
                if constexpr (kSum) us[t] = __ldg(a.dy2 + j);
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
                if constexpr (kSum) sum_grads(d, us[t]);
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
    if (threadIdx.x < kBnSlab)
        bn_bwd_channel<S>(tot, threadIdx.x, slab * kBnSlab + threadIdx.x, a.invstd, a.sum_dy, a.sum_dy_xhat, a.invstd2,
                          a.sum_dy2, a.sum_dy_xhat2);
}

struct BnBwdApplyArgs {
    const uint4* dy;
    const uint4* dy2;                // kSum only
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

template <int kUnroll, int kCtas, bool kShortcut, bool kSum>
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
        uint4 ud[kUnroll], ux[kUnroll], uy[kUnroll], u2[kShortcut ? kUnroll : 1], us[kSum ? kUnroll : 1];
        unsigned int mb[kUnroll];
#pragma unroll
        for (int t = 0; t < kUnroll; ++t) {
            const long long j = i + t * stride;
            ud[t] = ux[t] = uy[t] = make_uint4(0u, 0u, 0u, 0u);
            if constexpr (kShortcut) u2[t] = make_uint4(0u, 0u, 0u, 0u);
            if constexpr (kSum) us[t] = make_uint4(0u, 0u, 0u, 0u);
            mb[t] = 0u;
            if (j < a.V) {
                ud[t] = __ldg(a.dy + j);
                if constexpr (kSum) us[t] = __ldg(a.dy2 + j);
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
                if constexpr (kSum) sum_grads(d, us[t]);
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

void bn_stats_plan(long long M, int C, long long* passes, long long* ppc, int* R) {
    bn_reduce_plan(M, C, kBnStatsUnroll, kBnStatsCtas, passes, ppc, R);
}

void bn_bwd_reduce_plan(long long M, int C, long long* passes, long long* ppc, int* R) {
    bn_reduce_plan(M, C, kBnBwdReduceUnroll, kBnBwdReduceCtas, passes, ppc, R);
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
    return launched();
}
template <int U, int CT, bool SC>
static cudaError_t run_apply(BnApplyArgs& p, cudaStream_t stream) {
    bn_apply_kernel<U, CT, SC><<<bn_apply_grid(p.V, U, CT), kBnThreads, 0, stream>>>(p);
    return launched();
}
template <int U, int CT, bool SC, bool SUM = false>
static cudaError_t run_bwd_reduce(BnBwdReduceArgs& s, cudaStream_t stream) {
    bn_reduce_plan(s.M, s.C, U, CT, &s.passes, &s.ppc, &s.R);
    bn_bwd_reduce_kernel<U, CT, SC, SUM><<<dim3(s.C / kBnSlab, s.R), kBnThreads, 0, stream>>>(s);
    return launched();
}
template <int U, int CT, bool SC, bool SUM = false>
static cudaError_t run_bwd_apply(BnBwdApplyArgs& p, cudaStream_t stream) {
    bn_bwd_apply_kernel<U, CT, SC, SUM><<<bn_apply_grid(p.V, U, CT), kBnThreads, 0, stream>>>(p);
    return launched();
}

cudaError_t launch_bn_stats(const void* x, long long M, int C, const BnLayer& bn, void* ws, cudaStream_t stream) {
    if (!bn_shape_ok(M, C)) return cudaErrorNotSupported;
    BnStatsArgs s{};
    s.x = static_cast<const uint4*>(x);
    s.M = M; s.C = C;
    s.eps = bn.eps; s.momentum = bn.momentum;
    s.counters = static_cast<unsigned int*>(ws); s.partial = bn_ws_partials(ws);
    s.mean = bn.save_mean; s.invstd = bn.save_invstd;
    s.running_mean = bn.running_mean; s.running_var = bn.running_var; s.num_batches_tracked = bn.num_batches_tracked;
    return run_stats<kBnStatsUnroll, kBnStatsCtas>(s, stream);
}

cudaError_t launch_bn_fwd(const BnFwdPlan& f, cudaStream_t stream) {
    if (!bn_shape_ok(f.M, f.C)) return cudaErrorNotSupported;
    const BnLayer& bn = *f.bn;
    const BnLayer* sc = f.sc;
    cudaError_t e = cudaSuccess;
    if (!(f.given & MOCO_BN_STATS_GIVEN)) e = launch_bn_stats(f.x, f.M, f.C, bn, f.ws, stream);
    if (e == cudaSuccess && sc != nullptr && !(f.given & MOCO_BN_SC_STATS_GIVEN))
        e = launch_bn_stats(f.res, f.M, f.C, *sc, f.ws, stream);
    if (e != cudaSuccess) return e;
    BnApplyArgs p{};
    p.x = static_cast<const uint4*>(f.x); p.res = static_cast<const uint4*>(f.res); p.y = static_cast<uint4*>(f.y);
    p.mask = static_cast<uint8_t*>(f.mask);
    p.V = f.M * (f.C >> 3); p.C = f.C; p.relu = f.relu;
    p.mean = bn.save_mean; p.invstd = bn.save_invstd; p.gamma = bn.gamma; p.beta = bn.beta;
    if (sc == nullptr) return run_apply<kBnApplyUnroll, kBnApplyCtas, false>(p, stream);
    p.mean2 = sc->save_mean; p.invstd2 = sc->save_invstd; p.gamma2 = sc->gamma; p.beta2 = sc->beta;
    return run_apply<kBnApplyUnroll, kBnApplyCtas, true>(p, stream);
}

template <bool SUM>
static cudaError_t bwd_passes(BnBwdReduceArgs& s, BnBwdApplyArgs& p, bool shortcut, bool reduce, cudaStream_t stream) {
    cudaError_t e = cudaSuccess;
    if (reduce)
        e = shortcut ? run_bwd_reduce<kBnBwdReduceUnroll, kBnBwdReduceCtas, true, SUM>(s, stream)
                     : run_bwd_reduce<kBnBwdReduceUnroll, kBnBwdReduceCtas, false, SUM>(s, stream);
    if (e != cudaSuccess) return e;
    if (shortcut) return run_bwd_apply<kBnBwdApplyScUnroll, kBnBwdApplyScCtas, true, SUM>(p, stream);
    if constexpr (SUM) return run_bwd_apply<kBnBwdApplySumUnroll, kBnBwdApplySumCtas, false, true>(p, stream);
    return run_bwd_apply<kBnBwdApplyUnroll, kBnBwdApplyCtas, false, false>(p, stream);
}

cudaError_t launch_bn_bwd(const BnBwdPlan& b, cudaStream_t stream) {
    // apply only with a shortcut BN is not taken: its apply kernel reads the mask bits (kShortcut), and
    // moco_conv1x1_dgrad_bn_bwd does not produce a downsample block's g
    if (!bn_shape_ok(b.M, b.C) || (b.reduced && b.sc != nullptr)) return cudaErrorNotSupported;
    const int mask = b.mbits != nullptr ? kMaskFromBits
                                        : (!b.relu ? kMaskNone : (b.has_residual ? kMaskFromY : kMaskFromX));
    if (mask == kMaskFromY && b.y == nullptr) return cudaErrorInvalidValue;
    const BnLayer& bn = *b.bn;
    const BnLayer* sc = b.sc;
    BnBwdReduceArgs s{};
    s.dy = static_cast<const uint4*>(b.dy); s.dy2 = static_cast<const uint4*>(b.dy2); s.x = static_cast<const uint4*>(b.x);
    s.y = static_cast<const uint4*>(b.y); s.mbits = static_cast<const uint8_t*>(b.mbits);
    s.M = b.M; s.C = b.C; s.mask = mask;
    s.counters = static_cast<unsigned int*>(b.ws); s.partial = bn_ws_partials(b.ws);
    s.mean = bn.save_mean; s.invstd = bn.save_invstd; s.gamma = bn.gamma; s.beta = bn.beta;
    s.sum_dy = bn.dbeta; s.sum_dy_xhat = bn.dgamma;
    BnBwdApplyArgs p{};
    p.dy = s.dy; p.dy2 = s.dy2; p.x = s.x; p.y = s.y; p.mbits = s.mbits; p.dx = static_cast<uint4*>(b.dx);
    p.V = b.M * (b.C >> 3); p.C = b.C; p.mask = mask; p.inv_m = (float)(1.0 / (double)b.M);
    p.mean = bn.save_mean; p.invstd = bn.save_invstd; p.gamma = bn.gamma; p.beta = bn.beta;
    p.sum_dy = bn.dbeta; p.sum_dy_xhat = bn.dgamma;
    if (sc == nullptr) {
        p.dres = static_cast<uint4*>(b.dres);
    } else {
        s.x2 = p.x2 = static_cast<const uint4*>(b.x2);
        p.dx2 = static_cast<uint4*>(b.dres);
        s.mean2 = p.mean2 = sc->save_mean; s.invstd2 = p.invstd2 = sc->save_invstd;
        s.sum_dy2 = sc->dbeta; s.sum_dy_xhat2 = sc->dgamma;
        p.gamma2 = sc->gamma; p.sum_dy_xhat2 = sc->dgamma;
    }
    return b.dy2 != nullptr ? bwd_passes<true>(s, p, sc != nullptr, !b.reduced, stream)
                            : bwd_passes<false>(s, p, sc != nullptr, !b.reduced, stream);
}

cudaError_t launch_bn_relu_maxpool_fwd(const void* x, void* y, void* taps, int N, int H, int W, int C, const BnLayer& bn,
                                       void* ws, cudaStream_t stream) {
    if (N < 1 || H < 1 || W < 1) return cudaErrorNotSupported;
    cudaError_t e = launch_bn_stats(x, (long long)N * H * W, C, bn, ws, stream);
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
    return launched();
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
    return launched();
}

cudaError_t launch_bn_relu_maxpool_eval(const void* x, void* y, int N, int H, int W, int C, const float* scale,
                                        const float* shift, cudaStream_t stream) {
    if (N < 1 || H < 1 || W < 1 || !bn_shape_ok((long long)N * H * W, C)) return cudaErrorNotSupported;
    return launch_maxpool_fwd(x, y, nullptr, N, H, W, C, stream, nullptr, nullptr, nullptr, nullptr, scale, shift);
}

}  // namespace moco
