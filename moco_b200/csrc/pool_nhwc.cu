// 3x3 / stride 2 / pad 1 max pooling of the stem's channels_last bf16 activation (reference: moco/models/resnet.py:119,158
// `nn.MaxPool2d(kernel_size=3, stride=2, padding=1)`), forward and backward: one read of the input and one write of
// a quarter-size output.
//
// Semantics = torch.nn.functional.max_pool2d: out-of-image taps are skipped, the window is scanned kh then kw and
// the FIRST maximum wins (`val > max || isnan(val)`), which matters here because post-ReLU windows are full of equal
// zeros; the backward routes each output gradient to that one input element.  The forward stores the winner's tap
// number (0..8) as one byte per output element; the backward is a GATHER over the <= 4 windows that contain an input
// pixel (no atomics, deterministic, fp32 accumulation in increasing (oh, ow) order, one rounding to bf16).
//
// Both passes are HBM-bound.  Grid = (pixel tiles of one image, image): thread indices are 32-bit, the image offset is
// taken once per CTA, and the forward's per-channel BatchNorm coefficients are built once per CTA in shared memory.
//   forward   one thread per 16-byte vector (8 channels) of the output: 9 tap loads (neighbouring windows share
//             input vectors through L1 / L2), writes y (x/4 bytes) + 1 byte per output element
//   backward  one thread per output vector (oh, ow) and its 2x2 input quad (2oh..2oh+1, 2ow..2ow+1): the four windows
//             (oh..oh+1, ow..ow+1) that cover the quad are read once, each pixel takes the windows whose winning tap
//             is that pixel, and the quad's four dx vectors are written -- 4 window reads per 4 input pixels instead
//             of up to 4 per pixel.  With a second gradient (dy2, a block input's other branch) each window's
//             gradient is bf16(dy + dy2) before the gather, the value autograd's bf16 add would have stored.
#include "common.cuh"

#include <cuda_bf16.h>

namespace moco {

constexpr int kPoolThreads = 256;
constexpr int kPoolMaxCoefC = 2048;   // channels of the per-CTA coefficient table (the BatchNorm entry points' limit)

struct PoolArgs {
    const uint4* x;       // forward: input [N, H, W, C/8]; backward: dy [N, OH, OW, C/8]
    const uint4* x2;      // backward, nullable: dy2, added to dy
    uint4* y;             // forward: output [N, OH, OW, C/8]; backward: dx [N, H, W, C/8]
    uint2* idx;           // [N, OH, OW, C/8] x 8 tap bytes
    int N, H, W, OH, OW, lanes;
    int per_image;        // output vectors of one image: OH * OW * lanes
    int threads;          // threads per image: per_image (backward) or ceil(OH / 2) * ceil(OW / 2) * lanes (forward)
    // forward, nullable: the stem's BatchNorm + ReLU applied to every tap (rounded to bf16 as its own pass stores it)
    // before the max is taken -- the BatchNorm's output is never written
    const float* mean;
    const float* invstd;
    const float* gamma;
    const float* beta;
    // forward, nullable: a frozen BatchNorm's folded scale / shift applied to every tap by the header's eval contract
    // (moco_bn_relu_maxpool_eval); idx is then NULL
    const float* scale;
    const float* shift;
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

__device__ __forceinline__ uint4 pack8p(const float* f) {
    uint4 u;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
    for (int k = 0; k < 4; ++k) h[k] = __floats2bfloat162_rn(f[2 * k], f[2 * k + 1]);
    return u;
}

// relu(x * ca + cb + 0) rounded to bf16 as bn_apply_kernel stores it (kMode 1), bn_eval_kernel's relu(x * s + t) with
// no FMA (kMode 2), or x itself (kMode 0)
template <int kMode>
__device__ __forceinline__ void pool_tap8(const uint4& u, const float* ca, const float* cb, float* f) {
    unpack8p(u, f);
    if constexpr (kMode == 1) {
#pragma unroll
        for (int k = 0; k < 8; ++k)
            f[k] = __bfloat162float(__float2bfloat16_rn(fmaxf(__fadd_rn(fmaf(f[k], ca[k], cb[k]), 0.f), 0.f)));
    } else if constexpr (kMode == 2) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float z = __fadd_rn(__fmul_rn(f[k], ca[k]), cb[k]);
            f[k] = __bfloat162float(__float2bfloat16_rn(z > 0.f ? z : 0.f));
        }
    }
}

// kMode: 0 plain, 1 training BatchNorm + ReLU on every tap, 2 frozen BatchNorm + ReLU on every tap.
// One thread per 16-byte vector of a 2x2 tile of outputs (2th..2th+1, 2tw..2tw+1): the 5x5 input vectors under the
// tile are loaded row by row and taken through the BatchNorm once each (6.25 per output instead of 9), and every
// tap updates the outputs whose window holds it -- in row-major input order, which is each window's kh-then-kw order.
template <int kMode>
__global__ void __launch_bounds__(kPoolThreads)
maxpool3x3s2_fwd_kernel(const PoolArgs a) {
    extern __shared__ float4 coef_smem[];        // kMode != 0: ca[C], cb[C]
    float* sca = reinterpret_cast<float*>(coef_smem);
    float* scb = sca + a.lanes * 8;
    if constexpr (kMode != 0) {
        const int C = a.lanes * 8;
        for (int c = threadIdx.x; c < C; c += kPoolThreads) {
            if constexpr (kMode == 1) {
                const float ca = __ldg(a.gamma + c) * __ldg(a.invstd + c);
                sca[c] = ca;
                scb[c] = fmaf(-__ldg(a.mean + c), ca, __ldg(a.beta + c));
            } else {
                sca[c] = __ldg(a.scale + c);
                scb[c] = __ldg(a.shift + c);
            }
        }
        __syncthreads();
    }
    const int r = blockIdx.x * kPoolThreads + threadIdx.x;
    if (r >= a.threads) return;
    const int n = blockIdx.y;
    const int cv = r % a.lanes;
    const int p = r / a.lanes;
    const int TW = (a.OW + 1) >> 1;
    const int tw = p % TW, th = p / TW;
    const int ih0 = 4 * th - 1, iw0 = 4 * tw - 1;
    const uint4* x = a.x + (size_t)n * a.H * a.W * a.lanes + cv;
    float ca[8], cb[8];
    if constexpr (kMode != 0) {
        const float4* A = reinterpret_cast<const float4*>(sca + cv * 8);
        const float4* B = reinterpret_cast<const float4*>(scb + cv * 8);
        const float4 a0 = A[0], a1 = A[1], b0 = B[0], b1 = B[1];
        ca[0] = a0.x; ca[1] = a0.y; ca[2] = a0.z; ca[3] = a0.w; ca[4] = a1.x; ca[5] = a1.y; ca[6] = a1.z; ca[7] = a1.w;
        cb[0] = b0.x; cb[1] = b0.y; cb[2] = b0.z; cb[3] = b0.w; cb[4] = b1.x; cb[5] = b1.y; cb[6] = b1.z; cb[7] = b1.w;
    }
    // output o = 2i + j of the tile: running max and winning tap bytes (byte k of word k / 4)
    float m[4][8];
    unsigned int tw8[4][2];
    bool first[4];
#pragma unroll
    for (int o = 0; o < 4; ++o) {
        first[o] = true;
        tw8[o][0] = tw8[o][1] = 0u;
#pragma unroll
        for (int k = 0; k < 8; ++k) m[o][k] = -INFINITY;
    }
#pragma unroll
    for (int rr = 0; rr < 5; ++rr) {
        const int ih = ih0 + rr;
        if (ih < 0 || ih >= a.H) continue;
        uint4 u[5];
        unsigned int in = 0u;                    // bit c: column c lies inside the image
#pragma unroll
        for (int c = 0; c < 5; ++c) {
            const int iw = iw0 + c;
            const bool inside = iw >= 0 && iw < a.W;
            in |= (inside ? 1u : 0u) << c;
            u[c] = make_uint4(0u, 0u, 0u, 0u);
            if (inside) u[c] = __ldg(x + (ih * a.W + iw) * a.lanes);
        }
#pragma unroll
        for (int c = 0; c < 5; ++c) {
            if (!((in >> c) & 1u)) continue;
            float f[8];
            pool_tap8<kMode>(u[c], ca, cb, f);
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int kh = rr - 2 * i;
                if (kh < 0 || kh > 2) continue;
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int kw = c - 2 * j;
                    if (kw < 0 || kw > 2) continue;
                    const int o = 2 * i + j;
                    const unsigned int t = (unsigned int)(kh * 3 + kw);
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        // torch starts from the first in-image tap with max = -inf and replaces on
                        // `val > max || isnan(val)`; after the ReLU of kMode 1 / 2 no tap is NaN or below -0, so
                        // `val > max` alone is that rule there
                        const bool take = kMode == 0 ? (first[o] || f[k] > m[o][k] || f[k] != f[k]) : f[k] > m[o][k];
                        if (take) {
                            m[o][k] = f[k];
                            const int sh = 8 * (k & 3);
                            tw8[o][k >> 2] = (tw8[o][k >> 2] & ~(0xffu << sh)) | (t << sh);
                        }
                    }
                    first[o] = false;
                }
            }
        }
    }
    const size_t ybase = (size_t)n * a.per_image + cv;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int oh = 2 * th + i;
        if (oh >= a.OH) continue;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int ow = 2 * tw + j;
            if (ow >= a.OW) continue;
            const size_t o = ybase + (oh * a.OW + ow) * a.lanes;
            a.y[o] = pack8p(m[2 * i + j]);
            if (a.idx != nullptr) a.idx[o] = make_uint2(tw8[2 * i + j][0], tw8[2 * i + j][1]);   // NULL: eval
        }
    }
}

// acc[k] += g[k] where byte k of the window's tap bytes is `t`
__device__ __forceinline__ void gather_tap(float* acc, const float* g, const uint2& ix, unsigned int t) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const unsigned int tk = ((k < 4 ? ix.x : ix.y) >> (8 * (k & 3))) & 0xffu;
        if (tk == t) acc[k] += g[k];
    }
}

template <bool kSum>
__global__ void __launch_bounds__(kPoolThreads)
maxpool3x3s2_bwd_kernel(const PoolArgs a) {
    const int r = blockIdx.x * kPoolThreads + threadIdx.x;
    if (r >= a.threads) return;
    const int n = blockIdx.y;
    const int cv = r % a.lanes;
    const int p = r / a.lanes;
    const int ow = p % a.OW, oh = p / a.OW;
    const size_t obase = (size_t)n * a.per_image + cv;
    // windows w = 2 * dh + dw at (oh + dh, ow + dw); (oh, ow) always exists
    const bool right = ow + 1 < a.OW, down = oh + 1 < a.OH;
    const bool has[4] = {true, right, down, right && down};
    float g[4][8];
    uint2 ix[4];
#pragma unroll
    for (int w = 0; w < 4; ++w) {
        uint4 u = make_uint4(0u, 0u, 0u, 0u), u2 = make_uint4(0u, 0u, 0u, 0u);
        ix[w] = make_uint2(0u, 0u);
        if (has[w]) {
            const size_t o = obase + ((oh + (w >> 1)) * a.OW + ow + (w & 1)) * a.lanes;
            u = __ldg(a.x + o);
            if constexpr (kSum) u2 = __ldg(a.x2 + o);
            ix[w] = __ldg(a.idx + o);
        }
        unpack8p(u, g[w]);
        if constexpr (kSum) {
            float g2[8];
            unpack8p(u2, g2);
#pragma unroll
            for (int k = 0; k < 8; ++k) g[w][k] = __bfloat162float(__float2bfloat16_rn(__fadd_rn(g[w][k], g2[k])));
        }
    }
    // pixel (2oh + i, 2ow + j) is tap (1 + i - 2 dh) * 3 + (1 + j - 2 dw) of window (dh, dw); windows in (oh, ow) order
    const int h0 = 2 * oh, w0 = 2 * ow;
    uint4* dx = a.y + (size_t)n * a.H * a.W * a.lanes + cv;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    gather_tap(acc, g[0], ix[0], 4u);
    dx[(h0 * a.W + w0) * a.lanes] = pack8p(acc);
    const bool col1 = w0 + 1 < a.W, row1 = h0 + 1 < a.H;
    if (col1) {
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.f;
        gather_tap(acc, g[0], ix[0], 5u);
        if (right) gather_tap(acc, g[1], ix[1], 3u);
        dx[(h0 * a.W + w0 + 1) * a.lanes] = pack8p(acc);
    }
    if (row1) {
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.f;
        gather_tap(acc, g[0], ix[0], 7u);
        if (down) gather_tap(acc, g[2], ix[2], 1u);
        dx[((h0 + 1) * a.W + w0) * a.lanes] = pack8p(acc);
    }
    if (row1 && col1) {
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.f;
        gather_tap(acc, g[0], ix[0], 8u);
        if (right) gather_tap(acc, g[1], ix[1], 6u);
        if (down) gather_tap(acc, g[2], ix[2], 2u);
        if (right && down) gather_tap(acc, g[3], ix[3], 0u);
        dx[((h0 + 1) * a.W + w0 + 1) * a.lanes] = pack8p(acc);
    }
}

static bool pool_shape(int N, int H, int W, int C, PoolArgs* a) {
    if (N < 1 || H < 1 || W < 1 || C < 8 || (C & 7) != 0 || N > 65535) return false;
    a->N = N; a->H = H; a->W = W; a->lanes = C >> 3;
    a->OH = (H + 2 - 3) / 2 + 1;
    a->OW = (W + 2 - 3) / 2 + 1;
    // 32-bit indices within one image
    if ((long long)H * W * a->lanes > 0x7fffffffLL - kPoolThreads) return false;
    a->per_image = a->OH * a->OW * a->lanes;
    a->threads = a->per_image;
    return true;
}

static dim3 pool_grid(const PoolArgs& a) { return dim3((a.threads + kPoolThreads - 1) / kPoolThreads, a.N); }

cudaError_t launch_maxpool_fwd(const void* x, void* y, void* idx, int N, int H, int W, int C, cudaStream_t stream,
                               const float* bn_mean, const float* bn_invstd, const float* bn_gamma, const float* bn_beta,
                               const float* eval_scale, const float* eval_shift) {
    PoolArgs a{};
    if (!pool_shape(N, H, W, C, &a)) return cudaErrorNotSupported;
    a.x = static_cast<const uint4*>(x); a.y = static_cast<uint4*>(y); a.idx = static_cast<uint2*>(idx);
    a.mean = bn_mean; a.invstd = bn_invstd; a.gamma = bn_gamma; a.beta = bn_beta;
    a.scale = eval_scale; a.shift = eval_shift;
    a.threads = ((a.OH + 1) >> 1) * ((a.OW + 1) >> 1) * a.lanes;
    const bool bn = bn_gamma != nullptr, ev = eval_scale != nullptr;
    if ((bn || ev) && C > kPoolMaxCoefC) return cudaErrorNotSupported;
    const size_t smem = 2 * (size_t)C * sizeof(float);
    if (bn) maxpool3x3s2_fwd_kernel<1><<<pool_grid(a), kPoolThreads, smem, stream>>>(a);
    else if (ev) maxpool3x3s2_fwd_kernel<2><<<pool_grid(a), kPoolThreads, smem, stream>>>(a);
    else maxpool3x3s2_fwd_kernel<0><<<pool_grid(a), kPoolThreads, 0, stream>>>(a);
    return launched();
}

cudaError_t launch_maxpool_bwd(const void* dy, const void* dy2, const void* idx, void* dx, int N, int H, int W, int C,
                               cudaStream_t stream) {
    PoolArgs a{};
    if (!pool_shape(N, H, W, C, &a)) return cudaErrorNotSupported;
    a.x = static_cast<const uint4*>(dy); a.x2 = static_cast<const uint4*>(dy2); a.y = static_cast<uint4*>(dx);
    a.idx = const_cast<uint2*>(static_cast<const uint2*>(idx));
    if (dy2 != nullptr) maxpool3x3s2_bwd_kernel<true><<<pool_grid(a), kPoolThreads, 0, stream>>>(a);
    else maxpool3x3s2_bwd_kernel<false><<<pool_grid(a), kPoolThreads, 0, stream>>>(a);
    return launched();
}

}  // namespace moco
