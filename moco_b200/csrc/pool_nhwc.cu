// 3x3 / stride 2 / pad 1 max pooling of the stem's channels_last bf16 activation (reference: moco/models/resnet.py:119,158
// `nn.MaxPool2d(kernel_size=3, stride=2, padding=1)`), forward and backward: one read of the input and one write of
// a quarter-size output.
//
// Semantics = torch.nn.functional.max_pool2d: out-of-image taps are skipped, the window is scanned kh then kw and
// the FIRST maximum wins (`val > max || isnan(val)`), which matters here because post-ReLU windows are full of equal
// zeros; the backward routes each output gradient to that one input element.  The forward stores the winner's tap
// number (0..8) as one byte per output element; the backward is a GATHER over the <= 4 windows that contain an input
// pixel (no atomics, deterministic, fp32 accumulation, one rounding to bf16).
// One thread per 16-byte vector (8 channels) of the output (forward) / input (backward); HBM-bound:
//   forward   reads x once (neighbouring windows hit L1/L2), writes y (x/4 bytes) + 1 byte per output element
//   backward  reads dy + the tap bytes (each ~4x from cache), writes dx
#include "common.cuh"

#include <cuda_bf16.h>

namespace moco {

constexpr int kPoolThreads = 256;

struct PoolArgs {
    const uint4* x;       // forward: input [N, H, W, C/8]; backward: dy [N, OH, OW, C/8]
    uint4* y;             // forward: output [N, OH, OW, C/8]; backward: dx [N, H, W, C/8]
    uint2* idx;           // [N, OH, OW, C/8] x 8 tap bytes
    int N, H, W, OH, OW, lanes;
    long long total;      // vectors this launch produces
    // forward, nullable: the stem's BatchNorm + ReLU applied to every tap (rounded to bf16 as its own pass stores it)
    // before the max is taken -- the BatchNorm's output is never written
    const float* mean;
    const float* invstd;
    const float* gamma;
    const float* beta;
};

__device__ __forceinline__ void unpack8p(const uint4& u, float* f) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float2 t = __bfloat1622float2(h[k]);
        f[2 * k] = t.x;
        f[2 * k + 1] = t.y;
    }
}

__global__ void __launch_bounds__(kPoolThreads)
maxpool3x3s2_fwd_kernel(const PoolArgs a) {
    const long long o = (long long)blockIdx.x * kPoolThreads + threadIdx.x;
    if (o >= a.total) return;
    const int cv = (int)(o % a.lanes);
    long long p = o / a.lanes;
    const int ow = (int)(p % a.OW);
    p /= a.OW;
    const int oh = (int)(p % a.OH);
    const int n = (int)(p / a.OH);
    const bool bn = a.gamma != nullptr;
    float ca[8], cb[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        ca[k] = cb[k] = 0.f;
        if (bn) {
            const int c = cv * 8 + k;
            ca[k] = __ldg(a.gamma + c) * __ldg(a.invstd + c);
            cb[k] = fmaf(-__ldg(a.mean + c), ca[k], __ldg(a.beta + c));
        }
    }
    float m[8];
    unsigned int tap[8];
    bool first = true;
#pragma unroll
    for (int k = 0; k < 8; ++k) { m[k] = -INFINITY; tap[k] = 0u; }
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
        const int ih = 2 * oh - 1 + kh;
        if (ih < 0 || ih >= a.H) continue;
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
            const int iw = 2 * ow - 1 + kw;
            if (iw < 0 || iw >= a.W) continue;
            const uint4 u = __ldg(a.x + (((long long)n * a.H + ih) * a.W + iw) * a.lanes + cv);
            float f[8];
            unpack8p(u, f);
            if (bn) {
#pragma unroll
                for (int k = 0; k < 8; ++k)       // bn_apply_kernel's relu(x * ca + cb + 0), rounded to bf16
                    f[k] = __bfloat162float(__float2bfloat16_rn(fmaxf(__fadd_rn(fmaf(f[k], ca[k], cb[k]), 0.f), 0.f)));
            }
            const unsigned int t = (unsigned int)(kh * 3 + kw);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                // torch starts from the first in-image tap with max = -inf and replaces on `val > max || isnan(val)`
                if (first || f[k] > m[k] || f[k] != f[k]) { m[k] = f[k]; tap[k] = t; }
            }
            first = false;
        }
    }
    uint4 out;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&out);
#pragma unroll
    for (int k = 0; k < 4; ++k) h[k] = __floats2bfloat162_rn(m[2 * k], m[2 * k + 1]);
    a.y[o] = out;
    uint2 ix;
    ix.x = tap[0] | (tap[1] << 8) | (tap[2] << 16) | (tap[3] << 24);
    ix.y = tap[4] | (tap[5] << 8) | (tap[6] << 16) | (tap[7] << 24);
    a.idx[o] = ix;
}

__global__ void __launch_bounds__(kPoolThreads)
maxpool3x3s2_bwd_kernel(const PoolArgs a) {
    const long long i = (long long)blockIdx.x * kPoolThreads + threadIdx.x;
    if (i >= a.total) return;
    const int cv = (int)(i % a.lanes);
    long long p = i / a.lanes;
    const int w = (int)(p % a.W);
    p /= a.W;
    const int h = (int)(p % a.H);
    const int n = (int)(p / a.H);
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    // windows (oh, ow) with 2*oh - 1 <= h <= 2*oh + 1: oh in [ceil((h - 1) / 2), floor((h + 1) / 2)]
    const int oh0 = h >> 1, oh1 = (h + 1) >> 1;          // h even: {h/2}; h odd: {(h-1)/2, (h+1)/2}
    const int ow0 = w >> 1, ow1 = (w + 1) >> 1;
    for (int oh = oh0; oh <= oh1; ++oh) {
        if (oh >= a.OH) continue;
        const int kh = h - (2 * oh - 1);
        for (int ow = ow0; ow <= ow1; ++ow) {
            if (ow >= a.OW) continue;
            const int kw = w - (2 * ow - 1);
            const unsigned int t = (unsigned int)(kh * 3 + kw);
            const long long o = (((long long)n * a.OH + oh) * a.OW + ow) * a.lanes + cv;
            const uint2 ix = __ldg(a.idx + o);
            const uint4 u = __ldg(a.x + o);
            float g[8];
            unpack8p(u, g);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const unsigned int tk = ((k < 4 ? ix.x : ix.y) >> (8 * (k & 3))) & 0xffu;
                if (tk == t) acc[k] += g[k];
            }
        }
    }
    uint4 out;
    __nv_bfloat162* hh = reinterpret_cast<__nv_bfloat162*>(&out);
#pragma unroll
    for (int k = 0; k < 4; ++k) hh[k] = __floats2bfloat162_rn(acc[2 * k], acc[2 * k + 1]);
    a.y[i] = out;
}

static bool pool_shape(int N, int H, int W, int C, PoolArgs* a) {
    if (N < 1 || H < 1 || W < 1 || C < 8 || (C & 7) != 0) return false;
    a->N = N; a->H = H; a->W = W; a->lanes = C >> 3;
    a->OH = (H + 2 - 3) / 2 + 1;
    a->OW = (W + 2 - 3) / 2 + 1;
    return true;
}

cudaError_t launch_maxpool_fwd(const void* x, void* y, void* idx, int N, int H, int W, int C, cudaStream_t stream,
                               const float* bn_mean, const float* bn_invstd, const float* bn_gamma, const float* bn_beta) {
    PoolArgs a{};
    if (!pool_shape(N, H, W, C, &a)) return cudaErrorNotSupported;
    a.x = static_cast<const uint4*>(x); a.y = static_cast<uint4*>(y); a.idx = static_cast<uint2*>(idx);
    a.mean = bn_mean; a.invstd = bn_invstd; a.gamma = bn_gamma; a.beta = bn_beta;
    a.total = (long long)N * a.OH * a.OW * a.lanes;
    const long long blocks = (a.total + kPoolThreads - 1) / kPoolThreads;
    if (blocks > 0x7fffffffLL) return cudaErrorNotSupported;
    maxpool3x3s2_fwd_kernel<<<(unsigned int)blocks, kPoolThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_maxpool_bwd(const void* dy, const void* idx, void* dx, int N, int H, int W, int C, cudaStream_t stream) {
    PoolArgs a{};
    if (!pool_shape(N, H, W, C, &a)) return cudaErrorNotSupported;
    a.x = static_cast<const uint4*>(dy); a.y = static_cast<uint4*>(dx);
    a.idx = const_cast<uint2*>(static_cast<const uint2*>(idx));
    a.total = (long long)N * H * W * a.lanes;
    const long long blocks = (a.total + kPoolThreads - 1) / kPoolThreads;
    if (blocks > 0x7fffffffLL) return cudaErrorNotSupported;
    maxpool3x3s2_bwd_kernel<<<(unsigned int)blocks, kPoolThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

}  // namespace moco
