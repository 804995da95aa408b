// Weighted k-nearest-neighbour classification against a feature bank (moco_knn, include/moco_b200.h), without ever
// storing the [Nq, Nb] similarity matrix.
//
// s(i, j) = q_i . bank_j runs on the 1x1 convolutions' wgmma skeleton (conv1x1_skeleton.cuh): bank tiles of 128 rows
// are the GEMM's M, a CTA's column slice holds kKnnBN queries (N), C is the reduction (K-major B: q as stored).  The
// mainloop computes every tile's accumulator the same way in both sweeps, so the two see bit-identical similarities.
//
//   sweep 1 (knn_sweep_kernel<false>): the bank's tiles are taken in groups of kKnnGroup; warp w of the consumers sees
//     the same 16 rows of every tile, and its slice (g, w) is those rows over the tiles of group g.  The epilogue keeps
//     the running maximum of each query over the slice and writes it once: slice_max[q][8 g + w].  The slices are a
//     fixed partition of the bank (whole groups per CTA), so they do not depend on the grid.
//   threshold (knn_threshold_kernel): t_q = the k-th largest slice maximum.  k slices each hold a similarity >= t_q, so
//     t_q is at most the k-th largest similarity of q: every neighbour has s >= t_q.  With fewer than k non-empty
//     slices the k-th largest is -inf.
//   sweep 2 (knn_sweep_kernel<true>): the tiles again; every (s, j) with s >= t_q is appended to q's candidate list
//     through an atomic counter, as a 64-bit key whose order is the contract's (s descending, j ascending).  The list
//     order is not deterministic; what is in it is.
//   select (knn_select_kernel): one CTA per query.  A radix select finds the k-th largest key, the k keys at or above
//     it are sorted, and the vote runs over them in that order (the labels sorted by (label, rank), each class's
//     weights added by one thread in rank order).  The classes are ranked by (score descending, class ascending).
//
// A query with more candidates than the workspace holds is not truncated: the select kernel records the largest count
// and moco_knn reports it (MOCO_ERR_CAPACITY).
#include <cuda.h>
#include <cuda_bf16.h>
#include <math.h>

#include "../../include/moco_b200.h"
#include "common.cuh"
#include "conv1x1_skeleton.cuh"
#include "sm90_ptx.cuh"
#include "tc_common.cuh"

namespace moco {

constexpr int kKnnBN = 128;                // queries per CTA
constexpr int kKnnGroup = 8;               // tiles per slice group: a slice is 16 rows of each of them
constexpr int kKnnWarps = 8;               // consumer warps, one slice each per group
constexpr int kKnnSelThreads = 512;
constexpr int kKnnMaxK = 1024;

struct KnnArgs {
    int Nb, Nq, ksteps, m_tiles, groups, gpc, stages, n_slices;   // gpc = groups per CTA; ksteps = C / 64
    float* slice_max;                      // [Nq][n_slices]
    const float* thresh;                   // [Nq]
    unsigned int* count;                   // [Nq]
    unsigned long long* cand;              // [Nq][cap]
    unsigned int cap;
};

// A float's bits in an order where a larger key is a larger value; -0 is taken as +0.
__device__ __forceinline__ unsigned int knn_fkey(float s) {
    const unsigned int u = __float_as_uint(__fadd_rn(s, 0.f));
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float knn_fval(unsigned int k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
// (s descending, j ascending) as one descending 64-bit key
__device__ __forceinline__ unsigned long long knn_key(float s, int j) {
    return ((unsigned long long)knn_fkey(s) << 32) | (0xffffffffu - (unsigned int)j);
}

template <bool kPass2>
__global__ void __launch_bounds__(kCvThreads, 1)
knn_sweep_kernel(const __grid_constant__ CUtensorMap tm_bank, const __grid_constant__ CUtensorMap tm_q,
                 const KnnArgs a) {
    using S = Conv1x1Shape<kKnnBN>;
    extern __shared__ __align__(1024) uint8_t smem[];
    if ((smem_u32(smem) & 1023u) != 0u) __trap();
    const int NS = a.stages;
    uint8_t* ring = smem;                                          // NS x (bank slab, q slab)
    uint64_t* full = reinterpret_cast<uint64_t*>(ring + (size_t)NS * S::kStage);
    uint64_t* empty = full + NS;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nb = blockIdx.x;
    const int g0 = blockIdx.y * a.gpc;
    const int t0 = g0 * kKnnGroup;
    const int t1 = min(min(g0 + a.gpc, a.groups) * kKnnGroup, a.m_tiles);
    const int ksteps = a.ksteps;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm_bank);
        tma_prefetch_desc(&tm_q);
        for (int s = 0; s < NS; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp >= 8) {
        setmaxnreg_dec<40>();
        if (warp == 8 && elect_one()) {
            // ---------------------------------------------------- TMA producer
            int st = 0;
            uint32_t ph = 0;
            for (int tile = t0; tile < t1; ++tile)
                conv1x1_load_tile<kKnnBN, false>(&tm_bank, &tm_q, ring, full, empty, NS, st, ph, tile, nb, ksteps);
        }
        return;
    }
    // ------------------------------------------------------------ consumer warpgroups
    setmaxnreg_inc<232>();
    const int wg = warp >> 2, t = threadIdx.x & 127;
    const int rloc = wg * 64 + (warp & 3) * 16 + (lane >> 2);    // tile rows rloc and rloc + 8
    const int q0 = nb * kKnnBN + 2 * (lane & 3);                  // queries q0 + 8 j + e of acc[4 j + 2 h + e]
    float acc[kKnnBN / 2];
    float v[kKnnBN / 4];                                          // pass 1: running maxima; pass 2: thresholds
#pragma unroll
    for (int j = 0; j < kKnnBN / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int q = q0 + 8 * j + e;
            if constexpr (kPass2) v[2 * j + e] = q < a.Nq ? __ldg(a.thresh + q) : INFINITY;
            else                  v[2 * j + e] = -INFINITY;
        }
    int st = 0;
    uint32_t ph = 0;
    for (int tile = t0; tile < t1; ++tile) {
        conv1x1_mma_tile<kKnnBN, false>(acc, ring, wg, full, empty, NS, st, ph, ksteps, t);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = tile * kCvBM + rloc + 8 * h;
            if (row >= a.Nb) continue;                            // zero-filled rows past the bank
#pragma unroll
            for (int j = 0; j < kKnnBN / 8; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float s = acc[4 * j + 2 * h + e];
                    if constexpr (kPass2) {
                        if (s >= v[2 * j + e]) {                  // v = +inf past the queries
                            const int q = q0 + 8 * j + e;
                            const unsigned int pos = atomicAdd(a.count + q, 1u);
                            if (pos < a.cap) a.cand[(size_t)q * a.cap + pos] = knn_key(s, row);
                        }
                    } else {
                        v[2 * j + e] = fmaxf(v[2 * j + e], s);
                    }
                }
        }
        if constexpr (!kPass2) {
            if (tile % kKnnGroup == kKnnGroup - 1 || tile == a.m_tiles - 1) {   // the group's slices are complete
#pragma unroll
                for (int i = 0; i < kKnnBN / 4; ++i) {
                    float m = v[i];
                    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
                    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 8));
                    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 16));
                    const int q = q0 + 8 * (i >> 1) + (i & 1);
                    if (lane < 4 && q < a.Nq)
                        a.slice_max[(size_t)q * a.n_slices + (tile / kKnnGroup) * kKnnWarps + warp] = m;
                    v[i] = -INFINITY;
                }
            }
        }
    }
}

// The CTA's k-th largest of n keys load(i), exactly, by most-significant-digit radix select (8 bits per pass).
template <typename Key, typename Load>
__device__ Key radix_kth_largest(long long n, unsigned int k, Load load, unsigned int* hist, Key* sh_prefix,
                                 unsigned int* sh_k) {
    Key prefix = 0, mask = 0;
    unsigned int kk = k;
    for (int shift = (int)sizeof(Key) * 8 - 8; shift >= 0; shift -= 8) {
        for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        for (long long i = threadIdx.x; i < n; i += blockDim.x) {
            const Key key = load(i);
            if ((key & mask) == prefix) atomicAdd(&hist[(unsigned int)(key >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned int above = 0;
            int d = 255;
            for (; d > 0; --d) {
                if (above + hist[d] >= kk) break;
                above += hist[d];
            }
            *sh_prefix = prefix | ((Key)d << shift);
            *sh_k = kk - above;
        }
        __syncthreads();
        prefix = *sh_prefix;
        kk = *sh_k;
        mask |= (Key)255 << shift;
        __syncthreads();
    }
    return prefix;
}

// In-place bitonic sort of n (a power of two) smem elements by the CTA, descending.
template <typename T>
__device__ void bitonic_sort_desc(T* x, int n) {
    for (int size = 2; size <= n; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            __syncthreads();
            for (int i = threadIdx.x; i < n / 2; i += blockDim.x) {
                const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const T a = x[lo], b = x[hi];
                if (((lo & size) == 0) ? a < b : a > b) { x[lo] = b; x[hi] = a; }
            }
        }
    __syncthreads();
}

// t_q per query; also zeroes the candidate counters, the status words and the correct counts
__global__ void __launch_bounds__(256)
knn_threshold_kernel(const float* slice_max, int n_slices, int k, float* thresh, unsigned int* count,
                     unsigned int* status, int* correct) {
    __shared__ unsigned int hist[256];
    __shared__ unsigned int sh_prefix, sh_k;
    const int q = blockIdx.x;
    if (threadIdx.x == 0) {
        count[q] = 0;
        if (q == 0) {
            status[0] = status[1] = 0;
            if (correct != nullptr) correct[0] = correct[1] = 0;
        }
    }
    if (n_slices < k) {                                           // fewer slices than neighbours: every row
        if (threadIdx.x == 0) thresh[q] = -INFINITY;
        return;
    }
    const float* sm = slice_max + (size_t)q * n_slices;
    const unsigned int kth = radix_kth_largest<unsigned int>(
        n_slices, (unsigned int)k, [&](long long i) { return knn_fkey(sm[i]); }, hist, &sh_prefix, &sh_k);
    if (threadIdx.x == 0) thresh[q] = knn_fval(kth);
}

struct KnnSelectArgs {
    const int* labels;
    const int* targets;                    // nullable
    const unsigned int* count;
    const unsigned long long* cand;
    unsigned int cap;
    unsigned int* status;                  // [0] the largest count, [1] a label outside [0, n_classes)
    int k, n_classes;
    float inv_T;
    int* top5;                             // [Nq][5]
    float* scores5;                        // nullable [Nq][5]
    int* nbr_idx;                          // nullable [Nq][k]
    float* nbr_sim;                        // nullable [Nq][k]
    int* correct;                          // nullable [2]
};

__global__ void __launch_bounds__(kKnnSelThreads)
knn_select_kernel(const KnnSelectArgs a) {
    __shared__ unsigned long long key[kKnnMaxK];                  // the neighbours, then the classes' ranking keys
    __shared__ unsigned int lk[kKnnMaxK];                         // label << 10 | rank
    __shared__ float w[kKnnMaxK];                                 // the neighbours' weights by rank
    __shared__ unsigned int hist[256];
    __shared__ unsigned long long sh_prefix;
    __shared__ unsigned int sh_k, sh_n;
    const int q = blockIdx.x;
    const int k = a.k;
    const unsigned int m = a.count[q];
    if (threadIdx.x == 0) atomicMax(a.status, m);
    if (m > a.cap) return;                                        // the list was cut: compute nothing
    const unsigned long long* cq = a.cand + (size_t)q * a.cap;
    const unsigned long long kth = radix_kth_largest<unsigned long long>(
        m, (unsigned int)k, [&](long long i) { return cq[i]; }, hist, &sh_prefix, &sh_k);
    int P = 1;
    while (P < k) P <<= 1;
    for (int i = threadIdx.x; i < P; i += blockDim.x) key[i] = 0ull;   // below every key (j < 2^31)
    if (threadIdx.x == 0) sh_n = 0;
    __syncthreads();
    for (unsigned int i = threadIdx.x; i < m; i += blockDim.x) {        // exactly k keys: they are distinct
        const unsigned long long c = cq[i];
        if (c >= kth) key[atomicAdd(&sh_n, 1u)] = c;
    }
    bitonic_sort_desc(key, P);

    const float smax = knn_fval((unsigned int)(key[0] >> 32));
    for (int r = threadIdx.x; r < P; r += blockDim.x) {
        unsigned int l = 0xffffffffu;
        if (r < k) {
            const float s = knn_fval((unsigned int)(key[r] >> 32));
            const int j = (int)(0xffffffffu - (unsigned int)key[r]);
            if (a.nbr_idx != nullptr) a.nbr_idx[(size_t)q * k + r] = j;
            if (a.nbr_sim != nullptr) a.nbr_sim[(size_t)q * k + r] = s;
            int lab = __ldg(a.labels + j);
            if (lab < 0 || lab >= a.n_classes) { atomicOr(a.status + 1, 1u); lab = 0; }
            w[r] = expf(__fmul_rn(__fsub_rn(s, smax), a.inv_T));
            l = ((unsigned int)lab << 10) | (unsigned int)r;
        }
        lk[r] = ~l;                                               // descending sort of ~x: ascending (label, rank)
    }
    bitonic_sort_desc(lk, P);
    constexpr int kPer = kKnnMaxK / kKnnSelThreads;
    unsigned long long ck[kPer];                                  // the head of each label's run adds its weights
#pragma unroll
    for (int u = 0; u < kPer; ++u) {
        const int i = threadIdx.x + u * kKnnSelThreads;
        ck[u] = 0ull;
        if (i >= k) continue;
        const unsigned int l = ~lk[i];
        if (i > 0 && (~lk[i - 1]) >> 10 == l >> 10) continue;
        float score = 0.f;
        for (int r = i; r < k && (~lk[r]) >> 10 == l >> 10; ++r) score += w[(~lk[r]) & 1023u];
        ck[u] = ((unsigned long long)knn_fkey(score) << 32) | (0xffffffffu - (l >> 10));
    }
#pragma unroll
    for (int u = 0; u < kPer; ++u)                                // key[] is free: the neighbours were read above
        if (threadIdx.x + u * kKnnSelThreads < P) key[threadIdx.x + u * kKnnSelThreads] = ck[u];
    bitonic_sort_desc(key, P);
    if (threadIdx.x == 0) {
        int pred[5];
        float sc[5];
        int n = 0;
        for (int i = 0; i < 5 && i < k && key[i] != 0ull; ++i) {   // the classes with a positive score
            const float s = knn_fval((unsigned int)(key[i] >> 32));
            if (!(s > 0.f)) break;
            pred[n] = (int)(0xffffffffu - (unsigned int)key[i]);
            sc[n++] = s;
        }
        for (int c = 0; n < 5 && c < a.n_classes; ++c) {          // then score 0, by class
            bool taken = false;
            for (int i = 0; i < n; ++i) taken |= pred[i] == c;
            if (!taken) { pred[n] = c; sc[n++] = 0.f; }
        }
        for (; n < 5; ++n) { pred[n] = -1; sc[n] = 0.f; }         // fewer than 5 classes
        for (int i = 0; i < 5; ++i) {
            a.top5[q * 5 + i] = pred[i];
            if (a.scores5 != nullptr) a.scores5[q * 5 + i] = sc[i];
        }
        if (a.targets != nullptr && a.correct != nullptr) {
            const int tg = __ldg(a.targets + q);
            bool hit5 = false;
            for (int i = 0; i < 5; ++i) hit5 |= pred[i] == tg;
            if (pred[0] == tg) atomicAdd(a.correct, 1);
            if (hit5) atomicAdd(a.correct + 1, 1);
        }
    }
}

// ---- host side -------------------------------------------------------------------------------------------------
static long long knn_groups(long long Nb) { return ((Nb + kCvBM - 1) / kCvBM + kKnnGroup - 1) / kKnnGroup; }

KnnWorkspace knn_carve(void* base, int Nq, long long Nb, long long cap) {
    KnnWorkspace w;
    char* p = static_cast<char*>(base);
    size_t off = 0;
    w.n_slices = knn_groups(Nb) * kKnnWarps;
    w.status = reinterpret_cast<unsigned int*>(p + off);          off += 256;
    w.count = reinterpret_cast<unsigned int*>(p + off);           off += align_up((size_t)Nq * 4, 256);
    w.thresh = reinterpret_cast<float*>(p + off);                 off += align_up((size_t)Nq * 4, 256);
    w.slice_max = reinterpret_cast<float*>(p + off);              off += align_up((size_t)Nq * w.n_slices * 4, 256);
    w.cand = reinterpret_cast<unsigned long long*>(p + off);      off += (size_t)Nq * cap * 8;
    w.fixed = off - (size_t)Nq * cap * 8;
    w.cap = cap;
    w.bytes = off;
    return w;
}

bool knn_shape_ok(int Nq, long long Nb, int C, int k) {
    return Nq >= 1 && Nq <= kKnnMaxNq && C >= 64 && C <= 2048 && C % 64 == 0 && k >= 1 && k <= kKnnMaxK && Nb >= k &&
           Nb < (1LL << 31);
}

cudaError_t launch_knn(const void* q, const void* bank, const KnnPlan& p, const KnnWorkspace& ws, cudaStream_t stream) {
    using S = Conv1x1Shape<kKnnBN>;
    if (!knn_shape_ok(p.Nq, p.Nb, p.C, p.k) || ws.cap < (long long)p.k) return cudaErrorNotSupported;
    KnnArgs a{};
    a.Nb = (int)p.Nb; a.Nq = p.Nq; a.ksteps = p.C / 64;
    a.m_tiles = (int)((p.Nb + kCvBM - 1) / kCvBM);
    a.groups = (int)knn_groups(p.Nb);
    a.n_slices = (int)ws.n_slices;
    int dev = 0, sms = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return e;
    const int slices = (p.Nq + kKnnBN - 1) / kKnnBN;
    int R = sms / slices;                                  // one CTA per SM
    if (R < 1) R = 1;
    a.gpc = (a.groups + R - 1) / R;
    R = (a.groups + a.gpc - 1) / a.gpc;
    int smem = 0;
    e = ring_smem(0, S::kStage, &a.stages, &smem);
    if (e != cudaSuccess) return e;
    a.slice_max = ws.slice_max; a.thresh = ws.thresh; a.count = ws.count; a.cand = ws.cand;
    a.cap = (unsigned int)ws.cap;
    CUtensorMap tm_bank, tm_q;
    if (!make_tmap(&tm_bank, bank, (int)p.Nb, p.C, kCvBM) || !make_tmap(&tm_q, q, p.Nq, p.C, kKnnBN))
        return cudaErrorUnknown;
    e = launch_conv1x1<knn_sweep_kernel<false>>(dim3(slices, R), smem, stream, tm_bank, tm_q, a);
    if (e != cudaSuccess) return e;
    knn_threshold_kernel<<<p.Nq, 256, 0, stream>>>(ws.slice_max, a.n_slices, p.k, ws.thresh, ws.count, ws.status,
                                                   p.correct);
    e = launched();
    if (e != cudaSuccess) return e;
    e = launch_conv1x1<knn_sweep_kernel<true>>(dim3(slices, R), smem, stream, tm_bank, tm_q, a);
    if (e != cudaSuccess) return e;
    KnnSelectArgs s{};
    s.labels = p.labels; s.targets = p.targets; s.count = ws.count; s.cand = ws.cand; s.cap = a.cap;
    s.status = ws.status; s.k = p.k; s.n_classes = p.n_classes; s.inv_T = p.inv_T;
    s.top5 = p.top5; s.scores5 = p.scores5; s.nbr_idx = p.nbr_idx; s.nbr_sim = p.nbr_sim; s.correct = p.correct;
    knn_select_kernel<<<p.Nq, kKnnSelThreads, 0, stream>>>(s);
    return launched();
}

}  // namespace moco
