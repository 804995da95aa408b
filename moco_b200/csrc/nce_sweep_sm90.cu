// InfoNCE head on Hopper tensor cores (sm_90a): one persistent kernel sweeps a slice of the queue for a 128-row block
// of queries.  Three modes share it:
//
//   kFused  (one sweep, lse not known yet)   S = q . tile^T, P~ = 2^(S log2e/T - m), O~ += P~ . tile, l = sum P~
//   kNormed (two-pass dq, lse given)         the same with P = 2^(S log2e/T - lse log2e): O += P . tile
//   kStats  (two-pass statistics)            S = q . tile^T, online (max, sum 2^(x - max)) per row, optional dense
//                                            logits x = S / T
//
// Replaces torch.mm + cat + div + CrossEntropyLoss + softmax and autograd's backward GEMM with its queue clone
// (moco/NCE/Contrast.py:23-27, NCECriterion.py:11-13, train.py:264,273).
//
// Layout of the work.  384 threads: warps 0-3 and 4-7 are two consumer warpgroups, each owning 64 of the block's 128
// q rows; one thread of warp 8 is the TMA producer, and its warpgroup hands most of its registers to the consumers
// (setmaxnreg: 40 / 232 per thread).  q [N, C] is read by the consumers straight from the caller's tensor (fp32 or
// bf16, optionally L2-normalised here -- the reference's Normalize layer, moco/models/resnet.py:24-33 -- then rounded
// to bf16) and stored in the K-major 128-byte-swizzle layout wgmma reads: no separate cast kernel.  Queue tiles of BN
// rows (BN = 128 for C <= 128, 64 above, so that the O accumulator [64, C] and the S accumulator [64, BN] of a thread
// fit its registers together) are streamed by TMA through a ring of shared-memory stages.  Per tile a warpgroup runs
//   S[64, BN] = q . tile^T      wgmma, q and the tile from shared memory (both K-major)
//   P           softmax in registers; the S accumulator layout IS the register layout of wgmma's A operand, so P is
//               converted to bf16 pairs in place
//   O[64, C]  += P . tile       wgmma, P from registers, the SAME shared-memory tile as MN-major B
// and O stays in registers for the whole slice.  The stage goes back to the producer once both warpgroups' wgmmas
// on it have completed.
//
// Stabiliser (kFused): the CONSTANT m = log2e / T -- the largest logit a unit-norm query can have against a unit-norm
// queue row.  P~ = 2^(x - m), l = sum P~, O~ = sum P~ queue_j; the tail kernel (nce_tail.cu) merges the per-slice
// (m, l) pairs and rescales each slice's O~ by 2^(m - lse).  What can go wrong is only the exponent RANGE: rows far
// from unit norm.  The tail kernel detects both directions (a slice sum > 2^100, or a merged sum < 2^-80) and
// recomputes such rows exactly on CUDA cores, so the result equals the reference's for ANY q.
//
// CL = 2 (statistics mode, MOCO_NCE_CTA_PAIR): a cluster of two CTAs with different q blocks and the same queue
// slice; each CTA loads half of every queue tile and multicasts it into both, so the pair reads the slice from L2
// once.
#include <cuda.h>

#include "../../include/moco_b200.h"
#include "common.cuh"
#include "sm90_ptx.cuh"
#include "tc_common.cuh"

namespace moco {

constexpr int kFused = 0, kNormed = 1, kStats = 2;
constexpr int kSwThreads = 384;            // 2 consumer warpgroups + 1 producer warpgroup (one TMA thread)
constexpr int kQSlab = kRowsPerCta * 128;  // one [128 rows x 64 bf16] swizzled slab of q: 16 KB

struct SweepArgs {
    int N, C, K;
    int mblks, slices, n_pad, num_tiles, stages;
    float inv_T;
    const void* q;            // [N, C] fp32 or bf16 (q_dtype)
    int q_dtype;
    int normalize;            // 1: L2-normalise each q row before the bf16 rounding
    const float* lse;         // [N] natural log (kNormed)
    float* logits;            // optional dense [N, K+1] (kStats)
    float* part_o;            // [slices, n_pad, C]
    float2* part_ms;          // [slices, n_pad] (stabiliser, sum) in the log2 domain
    unsigned int* counters;   // workspace counters the tail kernel's last-block logic uses: zeroed here
    unsigned long long* cta_times;   // [grid][2] %globaltimer at entry / exit (profiling hook moco_prof_sweep_window)
};

template <int KC>
struct SweepShape {
    static constexpr int C = KC * 64;
    static constexpr int BN = KC <= 2 ? 128 : 64;        // queue rows per tile
    static constexpr int kTSlab = BN * 128;              // one [BN rows x 64 bf16] swizzled slab of a tile
    static constexpr int kTileBytes = KC * kTSlab;
    static constexpr int kQBytes = KC * kQSlab;
};

// q rows [64 wg, 64 wg + 64) of the block -> shared memory, K-major 128B-swizzle (row r at r * 128 B inside a 64-column
// slab, 16-byte chunk c at position c ^ (r & 7)).  A 16-byte piece of the source row per thread and step; the pieces
// of one row sit on consecutive lanes (a row is 8, 16 or 32 pieces when normalising), so its norm is a butterfly.
template <int KC>
__device__ __forceinline__ void stage_q(const SweepArgs& a, uint8_t* q_s, int row0, int wg, int t) {
    const int esz = (a.q_dtype == MOCO_F32) ? 4 : 2;
    const int cpr = KC * 64 * esz / 16;                   // 16-byte pieces per row
    const int total = 64 * cpr;
    for (int c = t; c < total; c += 128) {
        const int r = wg * 64 + c / cpr;
        const int piece = c - (c / cpr) * cpr;
        const int grow = row0 + r;
        const bool pad = grow >= a.N;
        const uint4 raw = __ldg(reinterpret_cast<const uint4*>(static_cast<const uint8_t*>(a.q) +
                                                             (size_t)(pad ? 0 : grow) * (KC * 64 * esz)) + piece);
        const int col0 = piece * (16 / esz);
        if (a.q_dtype == MOCO_F32) {                       // 4 fp32 -> 4 bf16 (8 bytes)
            float v0 = __uint_as_float(raw.x), v1 = __uint_as_float(raw.y);
            float v2 = __uint_as_float(raw.z), v3 = __uint_as_float(raw.w);
            if (a.normalize) {                             // x / sqrt(sum x^2): resnet.py:31-32
                float ss = v0 * v0 + v1 * v1 + v2 * v2 + v3 * v3;
                for (int w = cpr >> 1; w > 0; w >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, w);
                const float n = sqrtf(ss);
                v0 = v0 / n; v1 = v1 / n; v2 = v2 / n; v3 = v3 / n;
            }
            if (pad) { v0 = v1 = v2 = v3 = 0.f; }          // (0/0 of a padding row must not reach the MMA)
            const __nv_bfloat162 lo = __floats2bfloat162_rn(v0, v1), hi = __floats2bfloat162_rn(v2, v3);
            uint8_t* dst = q_s + (col0 >> 6) * kQSlab + sw128_offset(r, (col0 & 63) >> 3) + (col0 & 7) * 2;
            *reinterpret_cast<uint2*>(dst) = make_uint2(*reinterpret_cast<const uint32_t*>(&lo),
                                                        *reinterpret_cast<const uint32_t*>(&hi));
        } else {                                           // 8 bf16 = one 16-byte swizzle chunk
            uint4 u = raw;
            if (a.normalize) {
                float f[8];
                const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
                float ss = 0.f;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float2 x = __bfloat1622float2(h[e]);
                    f[2 * e] = x.x; f[2 * e + 1] = x.y;
                    ss = fmaf(x.x, x.x, fmaf(x.y, x.y, ss));
                }
                for (int w = cpr >> 1; w > 0; w >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, w);
                const float n = sqrtf(ss);
                __nv_bfloat162 o2[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) o2[e] = __floats2bfloat162_rn(f[2 * e] / n, f[2 * e + 1] / n);
                u = *reinterpret_cast<const uint4*>(o2);
            }
            if (pad) u = make_uint4(0u, 0u, 0u, 0u);
            uint8_t* dst = q_s + (col0 >> 6) * kQSlab + sw128_offset(r, (col0 & 63) >> 3);
            *reinterpret_cast<uint4*>(dst) = u;
        }
    }
}

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
    __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&h);
}

template <int KC, int MODE, int CL>
__global__ void __launch_bounds__(kSwThreads, 1)
nce_sweep_kernel(const __grid_constant__ CUtensorMap tm_queue, const SweepArgs a) {
    using S = SweepShape<KC>;
    constexpr int BN = S::BN;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw;
    if ((smem_u32(smem_raw) & 1023u) != 0u) __trap();
    // profiling hook (moco_prof_sweep_window): this slot is written by this kernel only and read by the host only, so the
    // store may precede griddepcontrol.wait
    if (threadIdx.x == 0 && a.cta_times != nullptr) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        a.cta_times[2 * blockIdx.x] = t;
    }
    const int NS = a.stages;
    uint8_t* q_s = smem;                                   // KC slabs of [128 rows x 128 B]
    uint8_t* v_s = q_s + S::kQBytes;                       // NS queue tiles
    uint64_t* bars = reinterpret_cast<uint64_t*>(v_s + (size_t)NS * S::kTileBytes);
    uint64_t* full = bars;
    uint64_t* empty = bars + NS;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t rank = (CL > 1) ? cluster_ctarank() : 0u;
    const int cluster_id = blockIdx.x / CL;
    const int mblk = cluster_id % a.mblks;
    const int slice = cluster_id / a.mblks;
    const int t0 = (int)(((long long)slice * a.num_tiles) / a.slices);
    const int t1 = (int)(((long long)(slice + 1) * a.num_tiles) / a.slices);
    const int ntiles = t1 - t0;
    const int row0 = (mblk * CL + (int)rank) * kRowsPerCta;

    pdl_launch_dependents();
    // ---- set-up that touches no global memory (overlaps the predecessor kernel under PDL) ----
    if (warp == 8 && lane == 0) {
        tma_prefetch_desc(&tm_queue);
        for (int s = 0; s < NS; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2 * CL); }
        fence_mbar_init();
    }
    if (CL > 1) cluster_sync_all(); else __syncthreads();
    pdl_wait();                                            // predecessor complete: q / lse / the queue are final
    if (blockIdx.x == 0 && threadIdx.x < 4 && a.counters != nullptr) a.counters[threadIdx.x] = 0u;

    if (warp >= 8) {
        setmaxnreg_dec<40>();
        if (warp == 8 && elect_one()) {
            // ------------------------------------------------ TMA producer (queue tiles)
            constexpr int kRowsPerLoad = BN / CL;
            int st = 0;
            uint32_t ph = 0;
            for (int i = 0; i < ntiles; ++i) {
                mbar_wait(&empty[st], ph ^ 1u);
                mbar_arrive_expect_tx(&full[st], (uint32_t)S::kTileBytes);
                uint8_t* dst = v_s + (size_t)st * S::kTileBytes + rank * (kRowsPerLoad * 128);
                const int brow = (t0 + i) * BN + (int)rank * kRowsPerLoad;
#pragma unroll
                for (int kc = 0; kc < KC; ++kc) {
                    if (CL > 1) tma_load_2d_mc(&tm_queue, &full[st], dst + kc * S::kTSlab, kc * 64, brow, (uint16_t)0x3);
                    else        tma_load_2d(&tm_queue, &full[st], dst + kc * S::kTSlab, kc * 64, brow);
                }
                if (++st == NS) { st = 0; ph ^= 1u; }
            }
        }
    } else {
        // ---------------------------------------------------- consumer warpgroups
        setmaxnreg_inc<232>();
        const int wg = warp >> 2;
        const int t = threadIdx.x & 127;
        stage_q<KC>(a, q_s, row0, wg, t);
        fence_proxy_async();                               // generic-proxy smem writes -> visible to wgmma
        named_bar_sync(1 + wg, 128);

        const int wrow = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // rows wrow and wrow + 8 of the block
        const int ccol = 2 * (lane & 3);                   // first of this thread's two columns in every 8-column group
        const float scale2 = a.inv_T * kLog2e;
        float lse2[2] = {scale2, scale2};                  // kFused: the stabiliser of unit-norm rows
        if (MODE == kNormed) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int g = row0 + wrow + 8 * h;
                lse2[h] = g < a.N ? a.lse[g] * kLog2e : 0.f;
            }
        }
        float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
        float* lrow[2] = {nullptr, nullptr};
        if (MODE == kStats && a.logits != nullptr) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int g = row0 + wrow + 8 * h;
                if (g < a.N) lrow[h] = a.logits + (size_t)g * (a.K + 1) + 1;
            }
        }

        const uint64_t q_desc = make_sw128_desc(smem_u32(q_s + wg * 64 * 128), 16, 1024);
        const uint64_t v_desc0 = make_sw128_desc(smem_u32(v_s), 16, 1024);                 // tile as K-major B
        const uint64_t vm_desc0 = make_sw128_desc(smem_u32(v_s), S::kTSlab, 1024);          // tile as MN-major B
        constexpr uint64_t kQSlabUnits = kQSlab >> 4, kTSlabUnits = S::kTSlab >> 4, kTileUnits = S::kTileBytes >> 4;
        float o[MODE == kStats ? 2 : KC * 32];
        int st = 0;
        uint32_t ph = 0;
        for (int i = 0; i < ntiles; ++i) {
            mbar_wait(&full[st], ph);
            float s[BN / 2];
            wgmma_fence();
#pragma unroll
            for (int kc = 0; kc < KC; ++kc)
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    wgmma_ss<BN>(s, q_desc + kc * kQSlabUnits + 2 * k, v_desc0 + st * kTileUnits + kc * kTSlabUnits + 2 * k,
                                 (kc | k) != 0);
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence(s);

            const int col0 = (t0 + i) * BN;
            const int valid = a.K - col0;                  // < BN on a ragged last tile only: columns >= K are TMA zeros
            if constexpr (MODE == kStats) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float cm = -INFINITY;
#pragma unroll
                    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                        for (int e = 0; e < 2; ++e)
                            if (valid >= BN || 8 * j + ccol + e < valid) cm = fmaxf(cm, s[4 * j + 2 * h + e]);
                    cm *= scale2;
                    if (cm > m[h]) { l[h] *= ex2(m[h] - cm); m[h] = cm; }
                    float acc = 0.f;
#pragma unroll
                    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int c = 8 * j + ccol + e;
                            if (valid >= BN || c < valid) {
                                acc += ex2(fmaf(s[4 * j + 2 * h + e], scale2, -m[h]));
                                if (lrow[h]) lrow[h][col0 + c] = s[4 * j + 2 * h + e] * a.inv_T;
                            }
                        }
                    l[h] += acc;
                }
            } else {
                uint32_t p[BN / 16][4];
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    float e4[4];
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            float x = ex2(fmaf(s[4 * j + 2 * h + e], scale2, -lse2[h]));
                            if (valid < BN && 8 * j + ccol + e >= valid) x = 0.f;   // also keeps inf * 0 out of O
                            e4[2 * h + e] = x;
                        }
                    if (MODE == kFused) { l[0] += e4[0] + e4[1]; l[1] += e4[2] + e4[3]; }
                    // A fragment of the 16-column step j / 2: {row h=0 cols 0-7, row h=1 cols 0-7, h=0 cols 8-15, h=1 8-15}
                    p[j >> 1][(j & 1) * 2 + 0] = pack_bf16(e4[0], e4[1]);
                    p[j >> 1][(j & 1) * 2 + 1] = pack_bf16(e4[2], e4[3]);
                }
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < BN / 16; ++kk)
                    wgmma_rs_tb<KC * 64>(o, p[kk], vm_desc0 + st * kTileUnits + kk * 128, (i | kk) != 0);
                wgmma_commit();
                wgmma_wait<0>();
                reg_fence(o);
            }
            // both warpgroups' wgmmas on this stage have completed once each leader arrived
            if (t == 0) {
                mbar_arrive(&empty[st]);
                if (CL > 1) mbar_arrive_cluster(&empty[st], rank ^ 1u);
            }
            if (++st == NS) { st = 0; ph ^= 1u; }
        }

        // ---- per-row results: the four threads of a quad hold one row's columns; merged in a fixed order
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = wrow + 8 * h;
            float2 ms;
            if (MODE == kStats) {
                float M = m[h];
                M = fmaxf(M, __shfl_xor_sync(0xffffffffu, M, 1));
                M = fmaxf(M, __shfl_xor_sync(0xffffffffu, M, 2));
                float L = (m[h] != -INFINITY) ? l[h] * ex2(m[h] - M) : 0.f;
                L += __shfl_xor_sync(0xffffffffu, L, 1);
                L += __shfl_xor_sync(0xffffffffu, L, 2);
                ms = make_float2(M, L);
            } else {
                float L = l[h];
                L += __shfl_xor_sync(0xffffffffu, L, 1);
                L += __shfl_xor_sync(0xffffffffu, L, 2);
                ms = make_float2(lse2[h], L);
            }
            if (MODE != kNormed && (lane & 3) == 0) a.part_ms[(size_t)slice * a.n_pad + row0 + r] = ms;
        }
        if constexpr (MODE != kStats) {
            // O epilogue: two consecutive columns per thread and 8-column group, streamed out (read once by the tail)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float* orow = a.part_o + ((size_t)slice * a.n_pad + row0 + wrow + 8 * h) * (KC * 64) + ccol;
#pragma unroll
                for (int j = 0; j < KC * 8; ++j)
                    __stcs(reinterpret_cast<float2*>(orow + 8 * j), make_float2(o[4 * j + 2 * h], o[4 * j + 2 * h + 1]));
            }
        }
    }

    if (CL > 1) cluster_sync_all(); else __syncthreads();  // no CTA of a pair leaves while its peer may still signal it
    if (threadIdx.x == 0 && a.cta_times != nullptr) {      // two plain stores per CTA; read by the bench's profiling hook
        unsigned long long t_exit;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_exit));
        a.cta_times[2 * blockIdx.x + 1] = t_exit;
    }
}

template <int KC, int MODE, int CL>
static cudaError_t launch_kc(const __nv_bfloat16* queue, SweepArgs& a, int* slices_out, cudaStream_t stream,
                             bool plan_only) {
    using S = SweepShape<KC>;
    a.num_tiles = (a.K + S::BN - 1) / S::BN;
    constexpr int kBarBytes = 256;
    int stages = (kSmemBudget - S::kQBytes - kBarBytes) / S::kTileBytes;
    if (stages > 8) stages = 8;
    if (stages < 2) return cudaErrorNotSupported;
    a.stages = stages;
    const int smem = S::kQBytes + stages * S::kTileBytes + kBarBytes;   // C = 128: 32 + 6 x 32 KB; C = 256: 64 + 5 x 32 KB
    CUtensorMap tm_queue = {};
    if (!plan_only && !make_tmap(&tm_queue, queue, a.K, KC * 64, S::BN / CL)) return cudaErrorUnknown;
    auto fill = [](SweepArgs& x, int slices) { x.slices = slices; };
    return plan_and_launch<nce_sweep_kernel<KC, MODE, CL>>(kSwThreads, smem, CL, a.mblks, a.mblks * CL, a.num_tiles,
                                                          a.n_pad, slices_out, stream, tm_queue, a, fill, true, plan_only);
}

template <int MODE, int CL>
static cudaError_t launch_mode(const __nv_bfloat16* queue, SweepArgs& a, int* slices_out, cudaStream_t stream,
                               bool plan_only) {
    switch (a.C) {
        case 64: return launch_kc<1, MODE, CL>(queue, a, slices_out, stream, plan_only);
        case 128: return launch_kc<2, MODE, CL>(queue, a, slices_out, stream, plan_only);
        case 192: return launch_kc<3, MODE, CL>(queue, a, slices_out, stream, plan_only);
        case 256: return launch_kc<4, MODE, CL>(queue, a, slices_out, stream, plan_only);
        default: return cudaErrorNotSupported;
    }
}

static SweepArgs sweep_args(const void* q, int q_dtype, int normalize, int N, int C, int K, float inv_T, int mblks,
                            int n_pad, const NceWorkspace& ws) {
    SweepArgs a;
    a.N = N; a.C = C; a.K = K;
    a.mblks = mblks; a.slices = 0; a.n_pad = n_pad; a.num_tiles = 0; a.stages = 0;
    a.inv_T = inv_T;
    a.q = q; a.q_dtype = q_dtype; a.normalize = normalize;
    a.lse = nullptr; a.logits = nullptr;
    a.part_o = ws.part_o;
    a.part_ms = ws.part_ms;
    a.counters = ws.counters;
    a.cta_times = ws.cta_times;
    return a;
}

bool nce_tc_shape_ok(int C) { return C % 64 == 0 && C >= 64 && C <= 256; }

// lse == nullptr selects the one-sweep mode (the kernel also writes ws.part_ms).
// plan_only: launch nothing, just report the slice count / padded rows this shape gets.
cudaError_t launch_nce_sweep(const void* q, int q_dtype, int normalize, const __nv_bfloat16* queue, int N, int C, int K,
                             float inv_T, const float* lse, int num_sms, int* slices_out, int* n_pad_out,
                             const NceWorkspace& ws, cudaStream_t stream, bool plan_only) {
    if (!nce_tc_shape_ok(C) || N < 1 || K < 1) return cudaErrorNotSupported;
    if (normalize && C > 128) return cudaErrorNotSupported;          // the in-kernel norm needs a row in one warp
    if ((reinterpret_cast<uintptr_t>(q) & 15) != 0) return cudaErrorNotSupported;
    const int mblks = (N + kRowsPerCta - 1) / kRowsPerCta;
    if (mblks > num_sms) return cudaErrorNotSupported;
    const int n_pad = mblks * kRowsPerCta;
    *n_pad_out = n_pad;
    SweepArgs a = sweep_args(q, q_dtype, normalize, N, C, K, inv_T, mblks, n_pad, ws);
    if (lse == nullptr) return launch_mode<kFused, 1>(queue, a, slices_out, stream, plan_only);
    a.lse = lse;
    return launch_mode<kNormed, 1>(queue, a, slices_out, stream, plan_only);
}

cudaError_t launch_nce_tc(NceTcParams& p, const NceWorkspace& ws, cudaStream_t stream) {
    if (!nce_tc_shape_ok(p.C) || p.N < 1 || p.K < 1) return cudaErrorNotSupported;
    const int G = p.cta_group;
    const int mblks = (p.N + kRowsPerCta * G - 1) / (kRowsPerCta * G);
    if (mblks * G > p.num_sms) return cudaErrorNotSupported;
    p.n_pad = mblks * G * kRowsPerCta;
    SweepArgs a = sweep_args(p.q_bf16, MOCO_BF16, 0, p.N, p.C, p.K, p.inv_T, mblks, p.n_pad, ws);
    a.logits = p.logits;
    if (G == 2) return launch_mode<kStats, 2>(p.queue, a, &p.slices, stream, false);
    return launch_mode<kStats, 1>(p.queue, a, &p.slices, stream, false);
}

}  // namespace moco
