// Tail of the one-sweep InfoNCE head: everything after the sweep kernel in ONE launch.
//
//   blocks [0, N)        one per query row: positive logit <q_i, k_i> (fp32, from the inputs as given, optionally
//                        L2-normalised here), merge of the per-slice (stabiliser, sum) pairs -> lse / loss_i / prob_i
//                        (NCESoftmaxLoss, moco/NCE/NCECriterion.py:11-13; `prob`, train.py:264), weighted sum of the
//                        per-slice O~ partials -> dq_i (autograd's result at train.py:273), and -- when the rows came
//                        in un-normalised -- the backward of the normalisation (Normalize, resnet.py:24-33):
//                        dx = (g - q^ <q^, g>) / |x|.
//   blocks [N, N + E)    FIFO enqueue of k_all (moco/NCE/Contrast.py:29-34), optionally normalising the key rows; the
//                        ring position comes by value or from a device int64 that the last block advances
//                        ((index + n_all) mod K, Contrast.py:34), which is what lets a captured CUDA graph replay.
//   last block           mean loss / mean prob in fixed order (no float atomics).
//
// The head kernel has finished before any block passes pdl_wait(), so the enqueue cannot disturb the logits of this
// step (the reference reads a clone for the same reason, Contrast.py:24-25).  The exact fallback below DOES read the
// queue inside this kernel, so the enqueue blocks load and convert their key rows first and then hold their stores
// until every row block has signalled that it is done with the queue (counters[1]; row blocks have the lower block
// indices and are dispatched first, so the wait cannot starve them; it is bounded and traps rather than hangs).
// This kernel WRITES the queue, so it never triggers its dependents early: the next kernel that reads the queue
// starts after it has completed.
//
// Exactness: the sweep kernel works with the constant exponent offset m = log2e/T for every row and every C (the
// largest logit of a unit-norm query against a unit-norm queue row).  If a slice's partial sum left the safe range
// (> 2^100: logits far above m) or the merged sum is so small that flushed terms could matter (< 2^-80 relative to
// the largest exponent: logits far below the bound, e.g. un-normalised q), the row falls back to the exact CUDA-core
// evaluation of that row against the whole queue (nce_rows.cuh): the one-sweep path is never silently wrong and never
// returns inf/NaN where the reference would not.  With L2-normalised features neither happens.
#include "../../include/moco_b200.h"
#include "common.cuh"
#include "nce_rows.cuh"
#include "sm90_ptx.cuh"

namespace moco {

constexpr int kTailThreads = kSimtThreads;         // 256
constexpr int kMaxTailDevices = 64;
constexpr int kTailMaxSlices = kMaxCtas;           // 160

struct TailArgs {
    int N, C, K, slices, n_pad;
    float inv_T;
    const void* q; const void* k; int qk_dtype; int normalize;
    const float2* part_ms; const float* part_o;
    float* lse; float* loss_rows; float* prob_rows; float* loss_prob; float* dq;
    unsigned int* counters;
    const __nv_bfloat16* queue;                    // pre-enqueue queue (exact fallback only)
    // enqueue (n_all == 0: none)
    __nv_bfloat16* enq_bf16; float* enq_f32; const void* k_all; int k_all_dtype; int n_all;
    long long index; long long* index_dev; long long row0, nrows;
    int enq_blocks;
};

__device__ __forceinline__ float block_sum_256(float v, float* red /*[8]*/) {
    v = warp_sum(v);
    __syncthreads();                                // protect `red` from the previous use
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < kTailThreads / 32; ++w) t += red[w];
    return t;
}

__global__ void __launch_bounds__(kTailThreads, 3)
nce_tail_kernel(const TailArgs a) {
    __shared__ SimtRowSmem sm;                     // exact fallback only (qs also serves as the q^ row)
    __shared__ float s_m[kTailMaxSlices];
    __shared__ float4 s_part[kTailThreads];
    __shared__ float s_red[8];
    __shared__ float s_val[4];                     // lse2, prob, unsafe flag
    pdl_wait();                                    // the head kernel has completed; see the header comment
    const int tid = threadIdx.x;
    const long long ring = a.index_dev ? *a.index_dev : a.index;
    if ((int)blockIdx.x < a.N) {
        const int i = blockIdx.x;
        const int C = a.C;
        const float scale2 = a.inv_T * kLog2e;
        // ---- q, k rows: <q, k>, |q|^2, |k|^2 (thread c owns elements c, c + 256, ...)
        float qe[kSimtMaxC / kTailThreads], ke[kSimtMaxC / kTailThreads];
        float dqk = 0.f, dqq = 0.f, dkk = 0.f;
#pragma unroll
        for (int u = 0; u < kSimtMaxC / kTailThreads; ++u) {
            const int c = tid + u * kTailThreads;
            qe[u] = ke[u] = 0.f;
            if (c < C) {
                qe[u] = load_as_float(a.q, a.qk_dtype, (size_t)i * C + c);
                ke[u] = load_as_float(a.k, a.qk_dtype, (size_t)i * C + c);
                dqk = fmaf(qe[u], ke[u], dqk); dqq = fmaf(qe[u], qe[u], dqq); dkk = fmaf(ke[u], ke[u], dkk);
            }
        }
        // prefetch this thread's share of the O~ partials while the statistics are merged
        const int lanes = C >> 2;
        const int groups = kTailThreads / lanes;           // C = 128: 8 groups of 32 float4 lanes
        const int lane4 = tid % lanes, grp = tid / lanes;
        constexpr int kPre = 10;
        float4 pre[kPre];
#pragma unroll
        for (int t = 0; t < kPre; ++t) {
            const int s = grp + t * groups;
            pre[t] = (grp < groups && s < a.slices)
                         ? __ldcs(reinterpret_cast<const float4*>(a.part_o + ((size_t)s * a.n_pad + i) * C) + lane4)
                         : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        // warp 0 also puts its (stabiliser, sum) pairs in flight now: one memory round trip for the whole block
        constexpr int kMsPre = (kTailMaxSlices + 31) / 32;     // 5
        float2 msr[kMsPre];
        if (tid < 32) {
#pragma unroll
            for (int t = 0; t < kMsPre; ++t) {
                const int s = tid + t * 32;
                msr[t] = (s < a.slices) ? a.part_ms[(size_t)s * a.n_pad + i] : make_float2(-INFINITY, 0.f);
            }
        }
        dqk = block_sum_256(dqk, s_red);
        float qn = 1.f, kn = 1.f;
        if (a.normalize) {
            dqq = block_sum_256(dqq, s_red);
            dkk = block_sum_256(dkk, s_red);
            qn = sqrtf(dqq); kn = sqrtf(dkk);
#pragma unroll
            for (int u = 0; u < kSimtMaxC / kTailThreads; ++u) { qe[u] = qe[u] / qn; ke[u] = ke[u] / kn; }
            dqk = dqk / (qn * kn);
        }
        const float lpos = dqk;
        const float x0 = lpos * scale2;
        // ---- merge the slices' (stabiliser, sum): warp 0
        if (tid < 32) {
            float m = x0, lmax = 0.f;
#pragma unroll
            for (int t = 0; t < kMsPre; ++t) {
                const int s = tid + t * 32;
                if (s < a.slices) {
                    s_m[s] = msr[t].x;
                    m = fmaxf(m, msr[t].x);
                    lmax = fmaxf(lmax, (msr[t].y == msr[t].y) ? msr[t].y : INFINITY);       // NaN counts as unsafe
                }
            }
            m = warp_max(m);
            lmax = warp_max(lmax);
            float l = 0.f;
#pragma unroll
            for (int t = 0; t < kMsPre; ++t)
                if (tid + t * 32 < a.slices) l += msr[t].y * ex2(msr[t].x - m);
            l = warp_sum(l);
            l += ex2(x0 - m);
            if (tid == 0) {
                s_val[0] = m + log2f(l);
                s_val[2] = (lmax > kOnePassUnsafeSum || !(l >= kOnePassUnderflow)) ? 1.f : 0.f;
            }
        }
        __syncthreads();
        float lse2 = s_val[0];
        const bool unsafe = s_val[2] != 0.f;
        float g[kSimtMaxC / kTailThreads];                // dL/dq^ for elements tid + u * 256
        float prob;
        if (!unsafe) {
            prob = exp2f(x0 - lse2);
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            if (grp < groups) {
#pragma unroll
                for (int t = 0; t < kPre; ++t) {
                    const int s = grp + t * groups;
                    if (s < a.slices) {
                        const float w = ex2(s_m[s] - lse2);
                        acc.x = fmaf(w, pre[t].x, acc.x); acc.y = fmaf(w, pre[t].y, acc.y);
                        acc.z = fmaf(w, pre[t].z, acc.z); acc.w = fmaf(w, pre[t].w, acc.w);
                    }
                }
                for (int s = grp + kPre * groups; s < a.slices; s += groups) {
                    const float4 v = __ldcs(reinterpret_cast<const float4*>(a.part_o + ((size_t)s * a.n_pad + i) * C) + lane4);
                    const float w = ex2(s_m[s] - lse2);
                    acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y);
                    acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
                }
                s_part[grp * lanes + lane4] = acc;
            }
            __syncthreads();
            // groups added in index order (deterministic); element c of the row sits in s_part[g * lanes + c / 4]
            const float gscale = a.inv_T / (float)a.N;
#pragma unroll
            for (int u = 0; u < kSimtMaxC / kTailThreads; ++u) {
                const int c = tid + u * kTailThreads;
                g[u] = 0.f;
                if (c < C) {
                    float t = 0.f;
                    for (int gi = 0; gi < groups; ++gi) t += reinterpret_cast<const float*>(&s_part[gi * lanes + (c >> 2)])[c & 3];
                    g[u] = gscale * (t + (prob - 1.f) * ke[u]);
                }
            }
        } else {
            // exact CUDA-core evaluation of this row (rare: see the header comment)
#pragma unroll
            for (int u = 0; u < kSimtMaxC / kTailThreads; ++u) {
                const int c = tid + u * kTailThreads;
                if (c < C) sm.qs[c] = __bfloat162float(__float2bfloat16_rn(qe[u]));
            }
            __syncthreads();
            lse2 = simt_row_stats(sm, lpos, a.queue, C, a.K, a.inv_T, nullptr);
            prob = exp2f(x0 - lse2);
            float acc[kSimtMaxC / kSimtThreads];
            simt_row_grad(sm, lse2, a.queue, C, a.K, a.inv_T, acc);
            const float gscale = a.inv_T / (float)a.N;
#pragma unroll
            for (int u = 0; u < kSimtMaxC / kTailThreads; ++u) g[u] = gscale * (acc[u] + (prob - 1.f) * ke[u]);
        }
        if (a.dq != nullptr) {
            if (a.normalize) {                            // through x -> x / |x|:  dx = (g - q^ <q^, g>) / |x|
                float dot = 0.f;
#pragma unroll
                for (int u = 0; u < kSimtMaxC / kTailThreads; ++u) dot = fmaf(qe[u], g[u], dot);
                dot = block_sum_256(dot, s_red);
#pragma unroll
                for (int u = 0; u < kSimtMaxC / kTailThreads; ++u) g[u] = (g[u] - qe[u] * dot) / qn;
            }
#pragma unroll
            for (int u = 0; u < kSimtMaxC / kTailThreads; ++u) {
                const int c = tid + u * kTailThreads;
                if (c < C) a.dq[(size_t)i * C + c] = g[u];
            }
        }
        if (tid == 0) {
            const float lse_nat = lse2 * kLn2;
            a.lse[i] = lse_nat;
            a.loss_rows[i] = lse_nat - lpos * a.inv_T;
            a.prob_rows[i] = prob;
        }
        if (a.n_all > 0) {                                // this block no longer reads the queue: release the enqueue
            __syncthreads();
            if (tid == 0) { __threadfence(); atomicAdd(a.counters + 1, 1u); }
        }
    } else if (a.n_all > 0) {
        // ---- enqueue blocks: queue[(ring + r) mod K] = k_all[r] (fp32 master + bf16 working copy), 8 elements per thread
        const int vec_per_row = a.C >> 3;
        const int rows_per_pass = kTailThreads / vec_per_row;
        const int v = tid % vec_per_row, rl = tid / vec_per_row;
        bool released = false;
        for (int r0 = ((int)blockIdx.x - a.N) * rows_per_pass; r0 < a.n_all; r0 += a.enq_blocks * rows_per_pass) {
            const int r = r0 + rl;
            const bool live = rl < rows_per_pass && r < a.n_all;
            float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            if (live) {
                if (a.k_all_dtype == MOCO_F32) {
                    const float4* src = reinterpret_cast<const float4*>(static_cast<const float*>(a.k_all) + (size_t)r * a.C) + v * 2;
                    const float4 x = src[0], y = src[1];
                    f[0] = x.x; f[1] = x.y; f[2] = x.z; f[3] = x.w; f[4] = y.x; f[5] = y.y; f[6] = y.z; f[7] = y.w;
                } else {
                    const uint4 u = *(reinterpret_cast<const uint4*>(static_cast<const __nv_bfloat16*>(a.k_all) + (size_t)r * a.C) + v);
                    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
                    for (int e = 0; e < 4; ++e) { const float2 x = __bfloat1622float2(h[e]); f[2 * e] = x.x; f[2 * e + 1] = x.y; }
                }
            }
            if (a.normalize) {                            // vec_per_row is a power of two <= 32 here (launcher)
                float ss = 0.f;
#pragma unroll
                for (int e = 0; e < 8; ++e) ss = fmaf(f[e], f[e], ss);
                for (int o = vec_per_row >> 1; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
                const float nrm = sqrtf(ss);
#pragma unroll
                for (int e = 0; e < 8; ++e) f[e] = f[e] / nrm;
            }
            if (!released) {                              // the first pass's rows are loaded and converted: now wait
                if (tid == 0) {
                    unsigned int seen, spins = 0;
                    do {
                        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(a.counters + 1) : "memory");
                        if (++spins > (1u << 26)) __trap();
                    } while (seen < (unsigned int)a.N);
                }
                __syncthreads();
                released = true;
            }
            if (live) {
                const long long dst = (ring + r) % a.K - a.row0;          // ring slot, relative to the rows this buffer holds
                if (dst >= 0 && dst < a.nrows) {
                    uint4 packed;
                    __nv_bfloat162* ph = reinterpret_cast<__nv_bfloat162*>(&packed);
#pragma unroll
                    for (int e = 0; e < 4; ++e) ph[e] = __floats2bfloat162_rn(f[2 * e], f[2 * e + 1]);
                    *(reinterpret_cast<uint4*>(a.enq_bf16 + (size_t)dst * a.C) + v) = packed;
                    if (a.enq_f32) {
                        float4* d = reinterpret_cast<float4*>(a.enq_f32 + (size_t)dst * a.C) + v * 2;
                        d[0] = make_float4(f[0], f[1], f[2], f[3]);
                        d[1] = make_float4(f[4], f[5], f[6], f[7]);
                    }
                }
            }
        }
    }
    const bool last = finish_mean(a.counters + 0, a.N, a.loss_rows, a.prob_rows, a.loss_prob);
    if (last && tid == 0) {
        a.counters[1] = 0u;                               // re-arm (every enqueue block has passed its wait: it arrived here)
        if (a.index_dev != nullptr && a.n_all > 0) *a.index_dev = (ring + a.n_all) % a.K;
    }
}

// can the tail kernel also do the enqueue for this shape?
bool nce_tail_can_enqueue(int C, int normalize) {
    if ((C & 7) != 0) return false;
    const int vec_per_row = C >> 3;
    if (vec_per_row > kTailThreads || kTailThreads % vec_per_row != 0) return false;
    if (normalize && ((vec_per_row & (vec_per_row - 1)) != 0 || vec_per_row > 32)) return false;
    return true;
}

// n_all == 0: no enqueue.  `normalize` applies to q, k and k_all alike.
cudaError_t launch_nce_tail(int N, int C, int K, int slices, int n_pad, float inv_T, const void* q, const void* k,
                            int qk_dtype, int normalize, const __nv_bfloat16* queue, float* lse, float* loss_rows,
                            float* prob_rows, float* loss_prob, float* dq, const NceWorkspace& ws,
                            __nv_bfloat16* enq_bf16, float* enq_f32, const void* k_all, int k_all_dtype, int n_all,
                            long long index, long long* index_dev, long long row0, long long nrows, cudaStream_t stream) {
    if ((C & 3) != 0 || C > kSimtMaxC || slices > kTailMaxSlices) return cudaErrorNotSupported;
    TailArgs a;
    a.N = N; a.C = C; a.K = K; a.slices = slices; a.n_pad = n_pad; a.inv_T = inv_T;
    a.q = q; a.k = k; a.qk_dtype = qk_dtype; a.normalize = normalize;
    a.part_ms = ws.part_ms; a.part_o = ws.part_o;
    a.lse = lse; a.loss_rows = loss_rows; a.prob_rows = prob_rows; a.loss_prob = loss_prob; a.dq = dq;
    a.counters = ws.counters;
    a.queue = queue;
    a.enq_bf16 = enq_bf16; a.enq_f32 = enq_f32; a.k_all = k_all; a.k_all_dtype = k_all_dtype; a.n_all = n_all;
    a.index = index; a.index_dev = index_dev; a.row0 = row0; a.nrows = nrows;
    a.enq_blocks = 0;
    if (n_all > 0) {
        const int vec_per_row = C >> 3;
        if (!nce_tail_can_enqueue(C, normalize)) return cudaErrorNotSupported;
        const int rows_per_pass = kTailThreads / vec_per_row;
        a.enq_blocks = (n_all + rows_per_pass - 1) / rows_per_pass;
        if (a.enq_blocks > 132) a.enq_blocks = 132;
    }
    // same shared-memory carve-out as the 227 KB head kernel in front of it: no SM reconfiguration between the two
    static bool carveout_set[kMaxTailDevices] = {false};
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && dev >= 0 && dev < kMaxTailDevices && !carveout_set[dev]) {
        cudaFuncSetAttribute(nce_tail_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        carveout_set[dev] = true;
    }
    return launch_pdl(nce_tail_kernel, dim3(N + a.enq_blocks), dim3(kTailThreads), 0, stream, a);
}


}  // namespace moco
