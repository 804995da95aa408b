// Support kernels of the InfoNCE head: prep (positive logit + bf16 cast of q),
// the cross-slice combine (lse / loss / prob / dq), the generic CUDA-core
// row kernel (any shape; also the on-GPU cross-check of the tensor-core kernels) and
// the dense-gradient backward of the compatibility API.
//
// Reference semantics: moco/NCE/Contrast.py:20-27, moco/NCE/NCECriterion.py:11-13,
// train.py:264,273 (see include/moco_b200.h).
#include "common.cuh"
#include "nce_rows.cuh"
#include "sm90_ptx.cuh"

namespace moco {

// ---------------------------------------------------------------------------
// prep: lpos[i] = <q_i, k_i> (fp32), q_bf16 = bf16(q) when q is fp32, zero counters.
// One warp per row.
// ---------------------------------------------------------------------------
__global__ void prep_kernel(const void* __restrict__ q, const void* __restrict__ k, int dtype, int N, int C,
                            float* __restrict__ lpos, __nv_bfloat16* __restrict__ q_bf16,
                            unsigned int* __restrict__ counters) {
    pdl_launch_dependents();
    pdl_wait();
    if (blockIdx.x == 0 && threadIdx.x < 4) counters[threadIdx.x] = 0u;
    int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= N) return;
    int lane = threadIdx.x & 31;
    float acc = 0.f;
    size_t base = (size_t)row * C;
    for (int c = lane; c < C; c += 32) {
        float qv = load_as_float(q, dtype, base + c);
        float kv = load_as_float(k, dtype, base + c);
        acc = fmaf(qv, kv, acc);
        if (dtype == 0) q_bf16[base + c] = __float2bfloat16_rn(qv);
    }
    acc = warp_sum(acc);
    if (lane == 0) lpos[row] = acc;
}

cudaError_t launch_prep(const void* q, const void* k, int qk_dtype, int N, int C, const NceWorkspace& ws,
                        cudaStream_t stream) {
    int rows_per_block = 4;
    return launch_pdl(prep_kernel, dim3((N + rows_per_block - 1) / rows_per_block), dim3(rows_per_block * 32), 0, stream,
                      q, k, qk_dtype, N, C, ws.lpos, ws.q_bf16, ws.counters);
}

// ---------------------------------------------------------------------------
// combine: merge the per-slice (max, sum[, O]) partials of the tensor-core kernel.
// One block per q row.
// ---------------------------------------------------------------------------
__global__ void combine_kernel(int N, int C, int K, int slices, int n_pad, float inv_T,
                               const float* __restrict__ lpos, const float2* __restrict__ part_ms,
                               float* __restrict__ logits,
                               float* __restrict__ lse, float* __restrict__ loss_rows,
                               float* __restrict__ prob_rows, float* __restrict__ loss_prob,
                               unsigned int* __restrict__ counters) {
    pdl_launch_dependents();
    pdl_wait();
    const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);     // one warp per q row
    const float scale2 = inv_T * kLog2e;
    if (i < N) {
        const float x0 = lpos[i] * scale2;         // positive logit, log2 domain
        int lane = threadIdx.x & 31;
        float m = x0;
        for (int s = lane; s < slices; s += 32) m = fmaxf(m, part_ms[(size_t)s * n_pad + i].x);
        m = warp_max(m);
        float l = 0.f;
        for (int s = lane; s < slices; s += 32) {
            float2 ms = part_ms[(size_t)s * n_pad + i];
            l += ms.y * ex2(ms.x - m);             // ms.x == -inf (empty slice) -> 0
        }
        l = warp_sum(l);
        l += ex2(x0 - m);
        float lse2 = m + log2f(l);
        if (lane == 0) {
            float lse_nat = lse2 * kLn2;
            float x0n = lpos[i] * inv_T;
            float prob = exp2f(x0 - lse2);
            lse[i] = lse_nat;
            loss_rows[i] = lse_nat - x0n;
            prob_rows[i] = prob;
            if (logits) logits[(size_t)i * (K + 1)] = x0n;
        }
    }
    finish_mean(counters + 0, N, loss_rows, prob_rows, loss_prob);
}

cudaError_t launch_combine(int N, int C, int slices, int n_pad, float inv_T, float* logits, int K, float* lse,
                           float* loss_rows, float* prob_rows, float* loss_prob, const NceWorkspace& ws,
                           cudaStream_t stream) {
    const int rows_per_block = 8;
    return launch_pdl(combine_kernel, dim3((N + rows_per_block - 1) / rows_per_block), dim3(rows_per_block * 32), 0,
                      stream, N, C, K, slices, n_pad, inv_T, ws.lpos, ws.part_ms, logits, lse, loss_rows, prob_rows,
                      loss_prob, ws.counters);
}

// Sharded queue, step 1: merge this rank's slices only -> one (max, sum) per row, no positive.  One warp per row.
// With ex.row_exact (one-sweep mode) a row whose sums left the one-sweep kernel's safe range is flagged there and
// evaluated exactly against the shard by the whole block: ms_out = (log2 of the shard's sum, 1).
constexpr int kPartialRows = 8;
static_assert(kPartialRows * 32 == kSimtThreads, "the exact evaluation takes the whole block");

__global__ void __launch_bounds__(kPartialRows * 32)
combine_partial_kernel(int N, int C, int slices, int n_pad, const float2* __restrict__ part_ms,
                       float2* __restrict__ ms_out, const ShardExact ex) {
    __shared__ SimtRowSmem sm;
    __shared__ int s_exact[kPartialRows];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * kPartialRows + w;
    bool exact = false;
    if (i < N) {
        float m = -INFINITY, lmax = 0.f;
        for (int s = lane; s < slices; s += 32) m = fmaxf(m, part_ms[(size_t)s * n_pad + i].x);
        m = warp_max(m);
        float l = 0.f;
        for (int s = lane; s < slices; s += 32) {
            float2 ms = part_ms[(size_t)s * n_pad + i];
            if (ms.x != -INFINITY) l += ms.y * ex2(ms.x - m);
            lmax = fmaxf(lmax, (ms.y == ms.y) ? ms.y : INFINITY);                // NaN counts as unsafe
        }
        l = warp_sum(l);
        if (ex.row_exact != nullptr) {
            lmax = warp_max(lmax);
            exact = lmax > kOnePassUnsafeSum || !(l >= kOnePassUnderflow);
            if (lane == 0) ex.row_exact[i] = exact ? 1 : 0;
        }
        if (lane == 0 && !exact) ms_out[i] = make_float2(m, l);
    }
    if (ex.row_exact == nullptr) return;
    if (lane == 0) s_exact[w] = exact ? 1 : 0;
    __syncthreads();
    for (int r = 0; r < kPartialRows; ++r) {                  // rare: the block's branch is uniform
        if (!s_exact[r]) continue;
        const int row = blockIdx.x * kPartialRows + r;
        for (int c = threadIdx.x; c < C; c += blockDim.x) sm.qs[c] = __bfloat162float(ex.q[(size_t)row * C + c]);
        __syncthreads();
        const float lse2 = simt_row_stats(sm, -INFINITY, ex.shard, C, ex.Ks, ex.inv_T, nullptr);
        if (threadIdx.x == 0) ms_out[row] = make_float2(lse2, 1.f);
        __syncthreads();                                      // sm is reused by the next flagged row
    }
}

cudaError_t launch_combine_partial(int N, int C, int slices, int n_pad, float2* ms_out, const NceWorkspace& ws,
                                   const ShardExact& exact, cudaStream_t stream) {
    if (exact.row_exact != nullptr && C > kSimtMaxC) return cudaErrorNotSupported;
    combine_partial_kernel<<<(N + kPartialRows - 1) / kPartialRows, kPartialRows * 32, 0, stream>>>(
        N, C, slices, n_pad, ws.part_ms, ms_out, exact);
    return launched();
}

// sharded queue, step 2: merge the W ranks' (max, sum) [W, N] with the positive logit (ws.lpos) -> lse, loss, prob
cudaError_t launch_combine_merge(int N, int world, float inv_T, const float2* ms_all, float* lse, float* loss_rows,
                                 float* prob_rows, float* loss_prob, const NceWorkspace& ws, cudaStream_t stream) {
    const int rows_per_block = 8;
    combine_kernel<<<(N + rows_per_block - 1) / rows_per_block, rows_per_block * 32, 0, stream>>>(
        N, 0, 0, world, N, inv_T, ws.lpos, ms_all, nullptr, lse, loss_rows, prob_rows, loss_prob, ws.counters);
    return launched();
}

// o_partial_i = sum_{j in shard} p_ij shard_j of one row, exactly (out of line: the common path keeps its registers)
__device__ __noinline__ void shard_exact_row_o(SimtRowSmem& sm, const __nv_bfloat16* __restrict__ q_row,
                                               const __nv_bfloat16* __restrict__ shard, int Ks, int C, float inv_T,
                                               float lse2, float* __restrict__ o_row) {
    for (int c = threadIdx.x; c < C; c += blockDim.x) sm.qs[c] = __bfloat162float(q_row[c]);
    __syncthreads();
    float acc[kSimtMaxC / kSimtThreads];
    simt_row_grad(sm, lse2, shard, C, Ks, inv_T, acc);
#pragma unroll
    for (int u = 0; u < kSimtMaxC / kSimtThreads; ++u) {
        const int c = threadIdx.x + u * kSimtThreads;
        if (c < C) o_row[c] = acc[u];
    }
}

// dq_i = inv_T / N * ( sum_slices w_s O_s[i] + (prob_i - 1) k_i )   -- fixed summation order.
// w_s = 1 when the dq kernel normalised with the final lse (two-pass); in one-pass mode slice s used its own
// stabiliser m_s (part_ms[s][i].x, log2 domain) and w_s = 2^(m_s - lse_i) finishes the normalisation here, except
// for the rows the sharded statistics call evaluated exactly (ex.row_exact): those are evaluated exactly here too.
__global__ void __launch_bounds__(kSimtThreads, 8)      // full occupancy: the exact branch is out of line
dq_reduce_kernel(int N, int C, int slices, int n_pad, float inv_T, const void* __restrict__ k,
                 int k_dtype, const float* __restrict__ part_o,
                 const float* __restrict__ prob_rows, float* __restrict__ dq,
                 const float2* __restrict__ part_ms, const float* __restrict__ lse, const ShardExact ex) {
    // 256 threads = (C/4 float4 lanes) x groups; group g sums slices g, g+groups, ...; groups are then
    // added in index order (deterministic).
    __shared__ union { float4 part[256]; SimtRowSmem row; } sh;
    float4* s_part = sh.part;
    pdl_launch_dependents();
    pdl_wait();
    const int i = blockIdx.x;
    if (ex.row_exact != nullptr && ex.row_exact[i]) {      // raw mode (o_partial), block-uniform branch
        shard_exact_row_o(sh.row, ex.q + (size_t)i * C, ex.shard, ex.Ks, C, ex.inv_T, lse[i] * kLog2e, dq + (size_t)i * C);
        return;
    }
    const int lanes = C >> 2;
    const int groups = 256 / lanes;
    const int lane = threadIdx.x % lanes, grp = threadIdx.x / lanes;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (grp < groups) {
        const float lse2 = part_ms ? lse[i] * kLog2e : 0.f;
        for (int s = grp; s < slices; s += groups) {
            float4 v = __ldcs(reinterpret_cast<const float4*>(part_o + ((size_t)s * n_pad + i) * C) + lane);
            if (part_ms) {
                const float w = ex2(part_ms[(size_t)s * n_pad + i].x - lse2);
                acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y);
                acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
            } else {
                acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
            }
        }
        s_part[grp * lanes + lane] = acc;
    }
    __syncthreads();
    if (grp == 0) {
        for (int g = 1; g < groups; ++g) {
            float4 v = s_part[g * lanes + lane];
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        const size_t base = (size_t)i * C + lane * 4;
        if (prob_rows == nullptr) {          // raw mode (sharded queue): just the slice sum
            *reinterpret_cast<float4*>(dq + base) = acc;
            return;
        }
        const float gscale = inv_T / (float)N;
        const float pm1 = prob_rows[i] - 1.f;
        float4 o;
        o.x = gscale * (acc.x + pm1 * load_as_float(k, k_dtype, base + 0));
        o.y = gscale * (acc.y + pm1 * load_as_float(k, k_dtype, base + 1));
        o.z = gscale * (acc.z + pm1 * load_as_float(k, k_dtype, base + 2));
        o.w = gscale * (acc.w + pm1 * load_as_float(k, k_dtype, base + 3));
        *reinterpret_cast<float4*>(dq + base) = o;
    }
}

cudaError_t launch_dq_reduce(int N, int C, int slices, int n_pad, float inv_T, const void* k, int k_dtype,
                             const float* prob_rows, float* dq, const float* part_o, cudaStream_t stream,
                             const float2* part_ms, const float* lse, const ShardExact& exact) {
    if ((C & 3) != 0 || C > 1024) return cudaErrorNotSupported;
    return launch_pdl(dq_reduce_kernel, dim3(N), dim3(kSimtThreads), 0, stream, N, C, slices, n_pad, inv_T, k, k_dtype,
                      part_o, prob_rows, dq, part_ms, lse, exact);
}

// Sharded queue, last step: dq_i = inv_T / N * ( sum_r O_r[row0 + i] + (prob_i - 1) k_i ), the W partial-gradient
// blocks O_r read straight from the peers' staging buffers over NVLink (replaces an NCCL reduce_scatter); ranks are
// summed in index order, so every run gives the same bits.  One block per row, C/4 float4 lanes.
struct PeerOTable { const float* base[16]; };

__global__ void dq_finish_peers_kernel(PeerOTable peers, int world, int row0, int N, int C, float inv_T,
                                       const void* __restrict__ k, int k_dtype, const float* __restrict__ prob_rows,
                                       float* __restrict__ dq) {
    const int i = blockIdx.x;
    const int lanes = C >> 2;
    for (int lane = threadIdx.x; lane < lanes; lane += blockDim.x) {
        float4 v[16];
#pragma unroll
        for (int r = 0; r < 16; ++r)                      // all peer loads in flight before the first add
            if (r < world) v[r] = __ldcv(reinterpret_cast<const float4*>(peers.base[r] + (size_t)(row0 + i) * C) + lane);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int r = 0; r < 16; ++r)
            if (r < world) { acc.x += v[r].x; acc.y += v[r].y; acc.z += v[r].z; acc.w += v[r].w; }
        const size_t base = (size_t)i * C + lane * 4;
        const float gscale = inv_T / (float)N;
        const float pm1 = prob_rows[i] - 1.f;
        float4 o;
        o.x = gscale * (acc.x + pm1 * load_as_float(k, k_dtype, base + 0));
        o.y = gscale * (acc.y + pm1 * load_as_float(k, k_dtype, base + 1));
        o.z = gscale * (acc.z + pm1 * load_as_float(k, k_dtype, base + 2));
        o.w = gscale * (acc.w + pm1 * load_as_float(k, k_dtype, base + 3));
        *reinterpret_cast<float4*>(dq + base) = o;
    }
}

cudaError_t launch_dq_finish_peers(const void* const* peers_host, int world, int rank, int N, int C, float inv_T,
                                   const void* k, int k_dtype, const float* prob_rows, float* dq, cudaStream_t stream) {
    if ((C & 3) != 0 || world < 1 || world > 16) return cudaErrorNotSupported;
    PeerOTable t;
    for (int r = 0; r < 16; ++r) t.base[r] = r < world ? static_cast<const float*>(peers_host[r]) : nullptr;
    int threads = C >> 2;
    if (threads > 256) threads = 256;
    if (threads < 32) threads = 32;
    dq_finish_peers_kernel<<<N, threads, 0, stream>>>(t, world, rank * N, N, C, inv_T, k, k_dtype, prob_rows, dq);
    return launched();
}

// ---------------------------------------------------------------------------
// Generic CUDA-core path: one block per q row, any (N, C <= 1024, K).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kSimtThreads)
simt_rows_kernel(const __nv_bfloat16* __restrict__ q_bf16, const void* __restrict__ k, int k_dtype,
                 const __nv_bfloat16* __restrict__ queue, int N, int C, int K, float inv_T,
                 const float* __restrict__ lpos, float* __restrict__ logits, float* __restrict__ lse,
                 float* __restrict__ loss_rows, float* __restrict__ prob_rows, float* __restrict__ loss_prob,
                 float* __restrict__ dq, unsigned int* __restrict__ counters) {
    __shared__ SimtRowSmem sm;
    const int i = blockIdx.x, tid = threadIdx.x;
    for (int c = tid; c < C; c += kSimtThreads) sm.qs[c] = __bfloat162float(q_bf16[(size_t)i * C + c]);
    __syncthreads();
    const float lse2 = simt_row_stats(sm, lpos[i], queue, C, K, inv_T, logits ? logits + (size_t)i * (K + 1) : nullptr);
    const float prob = exp2f(lpos[i] * inv_T * kLog2e - lse2);
    if (tid == 0) {
        const float lse_nat = lse2 * kLn2, x0n = lpos[i] * inv_T;
        lse[i] = lse_nat;
        loss_rows[i] = lse_nat - x0n;
        prob_rows[i] = prob;
    }
    if (dq) {
        float acc[kSimtMaxC / kSimtThreads];
        simt_row_grad(sm, lse2, queue, C, K, inv_T, acc);
        const float gscale = inv_T / (float)N;
#pragma unroll
        for (int u = 0; u < kSimtMaxC / kSimtThreads; ++u) {
            int c = tid + u * kSimtThreads;
            if (c < C) {
                float kv = load_as_float(k, k_dtype, (size_t)i * C + c);
                dq[(size_t)i * C + c] = gscale * (acc[u] + (prob - 1.f) * kv);
            }
        }
    }
    finish_mean(counters + 0, N, loss_rows, prob_rows, loss_prob);
}

cudaError_t launch_simt_rows(const __nv_bfloat16* q_bf16, const void* k, int k_dtype, const __nv_bfloat16* queue,
                             int N, int C, int K, float inv_T, float* logits, float* lse, float* loss_rows,
                             float* prob_rows, float* loss_prob, float* dq, const NceWorkspace& ws,
                             cudaStream_t stream) {
    if (C > kSimtMaxC) return cudaErrorNotSupported;
    simt_rows_kernel<<<N, kSimtThreads, 0, stream>>>(q_bf16, k, k_dtype, queue, N, C, K, inv_T, ws.lpos, logits,
                                                     lse, loss_rows, prob_rows, loss_prob, dq, ws.counters);
    return launched();
}

// ---------------------------------------------------------------------------
// Dense-gradient backward (compat API):  dq_i = inv_T (g_i0 k_i + sum_j g_i,1+j queue_j)
// kDenseRows q rows per block so the queue is streamed N / kDenseRows times.
// ---------------------------------------------------------------------------
constexpr int kDenseRows = 8;
constexpr int kDenseChunk = 128;

__global__ void __launch_bounds__(256)
bwd_dense_kernel(const float* __restrict__ g, const void* __restrict__ k, int k_dtype,
                 const __nv_bfloat16* __restrict__ queue, int N, int C, int K, float inv_T,
                 float* __restrict__ dq) {
    __shared__ float gs[kDenseRows][kDenseChunk];
    const int i0 = blockIdx.x * kDenseRows;
    const int c = blockIdx.y * blockDim.x + threadIdx.x;
    float acc[kDenseRows];
#pragma unroll
    for (int r = 0; r < kDenseRows; ++r) acc[r] = 0.f;
    for (int jb = 0; jb < K; jb += kDenseChunk) {
        for (int e = threadIdx.x; e < kDenseRows * kDenseChunk; e += blockDim.x) {
            int r = e / kDenseChunk, jj = e % kDenseChunk;
            int i = i0 + r, j = jb + jj;
            gs[r][jj] = (i < N && j < K) ? g[(size_t)i * (K + 1) + 1 + j] : 0.f;
        }
        __syncthreads();
        if (c < C) {
            int jn = min(kDenseChunk, K - jb);
            for (int jj = 0; jj < jn; ++jj) {
                float v = __bfloat162float(queue[(size_t)(jb + jj) * C + c]);
#pragma unroll
                for (int r = 0; r < kDenseRows; ++r) acc[r] = fmaf(gs[r][jj], v, acc[r]);
            }
        }
        __syncthreads();
    }
    if (c < C) {
#pragma unroll
        for (int r = 0; r < kDenseRows; ++r) {
            int i = i0 + r;
            if (i < N) {
                float kv = load_as_float(k, k_dtype, (size_t)i * C + c);
                dq[(size_t)i * C + c] = inv_T * (g[(size_t)i * (K + 1)] * kv + acc[r]);
            }
        }
    }
}

cudaError_t launch_bwd_dense(const float* g, const void* k, int k_dtype, const __nv_bfloat16* queue, int N, int C,
                             int K, float inv_T, float* dq, cudaStream_t stream) {
    int threads = C >= 256 ? 256 : ((C + 31) / 32 * 32);
    dim3 grid((N + kDenseRows - 1) / kDenseRows, (C + threads - 1) / threads);
    bwd_dense_kernel<<<grid, threads, 0, stream>>>(g, k, k_dtype, queue, N, C, K, inv_T, dq);
    return launched();
}

}  // namespace moco
