// Momentum (EMA) update of the key encoder as ONE multi-tensor launch.
//
// Reference: moco/util.py:124-127 (called at train.py:277 every step, and once with m = 0 at train.py:133):
//     for p1, p2 in zip(model.parameters(), model_ema.parameters()):
//         p2.data.mul_(m).add_(1 - m, p1.detach().data)
// i.e. per element   t = rn(p2 * m);  p2 = fma(1 - m, p1, t)   (ATen's add-with-alpha contracts to an FMA on
// both its CUDA and its vectorised CPU path), which is exactly what the kernel evaluates -- bit-exact with the
// reference's two passes, in one pass: 322 tiny launches (ResNet-50: 161 tensors x 2 ops) become one, and the
// EMA weights are read once and written once (12 B/element of HBM traffic instead of 20).
//
// Work decomposition: the host describes the tensors as a DEVICE table of segments {p_ema, p, n} plus an
// exclusive prefix of per-segment chunk counts; block b walks chunks b, b + grid, ... and locates its segment by
// binary search in the prefix (<= 8 probes for a ResNet, L1/L2 resident).  HBM-bound: each thread keeps
// 2 x kUnroll 16-byte loads in flight.
#include "common.cuh"

namespace moco {

struct EmaSeg {
    float* p_ema;
    const float* p;
    long long n;
};
static_assert(sizeof(EmaSeg) == 24, "EmaSeg is three 64-bit words (int64 [n_segs, 3] on the host side)");

constexpr int kEmaThreads = 256;
constexpr int kEmaUnroll = 4;
constexpr int kEmaChunk = kEmaThreads * 4 * kEmaUnroll * 2;   // 8192 elements = 32 KB per operand per chunk

__device__ __forceinline__ float ema_one(float pe, float p, float m, float one_minus_m) {
    return __fmaf_rn(one_minus_m, p, __fmul_rn(pe, m));
}

__global__ void __launch_bounds__(kEmaThreads)
ema_multi_kernel(const EmaSeg* __restrict__ segs, const int* __restrict__ chunk_prefix, int n_segs, int n_chunks,
                 float m, float one_minus_m) {
    for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
        // segment s with chunk_prefix[s] <= c < chunk_prefix[s + 1]
        int lo = 0, hi = n_segs;
        while (hi - lo > 1) {
            int mid = (lo + hi) >> 1;
            if (__ldg(chunk_prefix + mid) <= c) lo = mid; else hi = mid;
        }
        const EmaSeg sg = segs[lo];
        const long long start = (long long)(c - __ldg(chunk_prefix + lo)) * kEmaChunk;
        long long left = sg.n - start;
        const int cnt = left < kEmaChunk ? (int)left : kEmaChunk;
        float* pe = sg.p_ema + start;
        const float* p = sg.p + start;
        const bool vec = (((uintptr_t)pe | (uintptr_t)p) & 15) == 0;
        if (vec && cnt == kEmaChunk) {
            float4* pe4 = reinterpret_cast<float4*>(pe);
            const float4* p4 = reinterpret_cast<const float4*>(p);
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                float4 a[kEmaUnroll], b[kEmaUnroll];
#pragma unroll
                for (int u = 0; u < kEmaUnroll; ++u) {
                    int i = (half * kEmaUnroll + u) * kEmaThreads + threadIdx.x;
                    a[u] = pe4[i];
                    b[u] = __ldg(p4 + i);
                }
#pragma unroll
                for (int u = 0; u < kEmaUnroll; ++u) {
                    int i = (half * kEmaUnroll + u) * kEmaThreads + threadIdx.x;
                    float4 r;
                    r.x = ema_one(a[u].x, b[u].x, m, one_minus_m);
                    r.y = ema_one(a[u].y, b[u].y, m, one_minus_m);
                    r.z = ema_one(a[u].z, b[u].z, m, one_minus_m);
                    r.w = ema_one(a[u].w, b[u].w, m, one_minus_m);
                    pe4[i] = r;
                }
            }
        } else if (vec) {
            const int n4 = cnt >> 2;
            float4* pe4 = reinterpret_cast<float4*>(pe);
            const float4* p4 = reinterpret_cast<const float4*>(p);
            for (int i = threadIdx.x; i < n4; i += kEmaThreads) {
                float4 a = pe4[i], b = __ldg(p4 + i), r;
                r.x = ema_one(a.x, b.x, m, one_minus_m);
                r.y = ema_one(a.y, b.y, m, one_minus_m);
                r.z = ema_one(a.z, b.z, m, one_minus_m);
                r.w = ema_one(a.w, b.w, m, one_minus_m);
                pe4[i] = r;
            }
            for (int i = (n4 << 2) + threadIdx.x; i < cnt; i += kEmaThreads) pe[i] = ema_one(pe[i], p[i], m, one_minus_m);
        } else {
            for (int i = threadIdx.x; i < cnt; i += kEmaThreads) pe[i] = ema_one(pe[i], p[i], m, one_minus_m);
        }
    }
}

int ema_chunk_elems() { return kEmaChunk; }

cudaError_t launch_ema(const void* segs, const int* chunk_prefix, int n_segs, int n_chunks, float m, float one_minus_m,
                       cudaStream_t stream) {
    if (n_segs == 0 || n_chunks == 0) return cudaSuccess;
    int blocks = n_chunks < 132 * 8 ? n_chunks : 132 * 8;
    ema_multi_kernel<<<blocks, kEmaThreads, 0, stream>>>(static_cast<const EmaSeg*>(segs), chunk_prefix, n_segs, n_chunks,
                                                         m, one_minus_m);
    return launched();
}

}  // namespace moco
