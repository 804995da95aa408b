// The bottleneck blocks' 1x1 convolutions on Hopper tensor cores (sm_90a), with BatchNorm work in their epilogues.
// In NHWC a 1x1 / stride 1 convolution is a GEMM over the M = N*H*W pixel rows (bf16 operands, fp32 accumulation, each
// output rounded to bf16 once).  Its three kernels share one skeleton (conv1x1_skeleton.cuh, which the kNN similarity
// sweep of knn_sm90.cu runs too).
//
// 384 threads: warps 0-3 and 4-7 are two consumer warpgroups, each owning 64 rows of the CTA's 128-row tile; one
// thread of warp 8 is the TMA producer (setmaxnreg: 40 / 232 registers per thread).  A CTA owns one BN-column slice of
// the output and a contiguous range of 128-row tiles.  Per tile and 64-wide K chunk the producer loads the A slab
// [128 x 64] and the B slab (BN columns x 64) into a ring of smem stages; each warpgroup runs wgmma m64nBNk16 x 4 from
// smem (A K-major, B K-major or MN-major, 128-byte swizzle) in increasing K, so every kernel that runs the mainloop
// computes the same accumulator for the same tile.  The epilogue rounds the accumulator to bf16, stages it in smem in
// the swizzled layout and stores it with TMA bulk stores.  A kernel whose epilogue reads operands other than the
// accumulator has the producer load them into two buffers, one tile ahead of the consumers.  The BatchNorm reductions
// read the staged bf16 tile back in the thread layout and fp32 order of the BatchNorm kernel they replace (bn_nhwc.cu),
// and its per-CTA partials and fixed-order fp64 finish in the last CTA of a slab (bn_reduce.cuh) run on the consumers'
// named barriers: bit-identical results.
//
// conv1x1_stats_kernel: y[M, Cout] = x[M, Cin] . w[Cout, Cin]^T for conv1 -> bn1, conv3 -> bn3 and the stride-1
// shortcut -> BatchNorm (moco/models/resnet.py:74-102,139-143), with the batch statistics of y AS ROUNDED to bf16, the
// tensor the BatchNorm reads.  They replace that BatchNorm's statistics pass (bn_stats_kernel), which would read y back
// from HBM once more.  BN = 128, or 64 when Cout is not a multiple of 128.  Each warpgroup stages its 64 rows in a
// double-buffered tile of its own and stores them with one TMA store per 64 columns.  The row ranges of the CTAs are
// those of the statistics pass (bn_stats_plan: a chunk is a multiple of 256 rows, so whole tiles); thread (v, rl) takes
// channels 8v .. 8v+7 of each 64-channel slab in rows rl, rl + 32, ... in increasing order and adds (y - y[0, c]) and
// its square.  y[0, c], the shift, is computed by every CTA: the CTAs after the first run tile 0 once more, without
// storing it.
//
// conv1x1_bn_apply_kernel: the residual BatchNorm applied in a second pass of the GEMM.  Once the statistics of
// h = x . w^T are known (the kernel above), the block output y = relu(bn(h) + r) is computed from x again rather than
// from h read back: for conv3 of a bottleneck (K = Cin = Cout / 4) the GEMM costs less than the 8 bytes per element of
// h written and read.  The mainloop has the same BN as the statistics pass, so the accumulator of a tile is the one it
// rounded.  The epilogue is bn_apply_kernel's arithmetic (bn_nhwc.cu): h rounded to bf16, z = fmaf(h, ca, cb) + r with
// ca = gamma * invstd, cb = fmaf(-mean, ca, beta), ReLU, one rounding; with a shortcut BN r = bf16(fmaf(s, ca2, cb2) +
// 0) of the shortcut convolution's raw output s.  The mask bytes (nullable) are relu_bits of the staged output.  The
// epilogue operand is the r (or s) tile; y is staged in place over it and stored from there.  The grid is one wave: a
// column slice per blockIdx.x, contiguous tile ranges per blockIdx.y.
//
// conv1x1_dgrad_bn_bwd_kernel: the input gradient with the producing BatchNorm's backward reduction.  The convolution's
// input is the output of a block's residual BatchNorm, y = relu(bn(x) + r), and it has a second consumer, the next
// block's residual branch, whose gradient dy2 is handed over (bn.py: hand_over).  The dgrad GEMM
//     dX[M, Cin] = dH[M, Cout] . w[Cout, Cin]                 (w as stored is the MN-major B operand)
// rounds dX to bf16 (what cuDNN's dgrad stores), adds dy2 with sum_grads' single rounding and applies the forward's
// ReLU mask bits: g, the masked gradient that bn_bwd_reduce_kernel / bn_bwd_apply_kernel would form from the same
// inputs.  g is written once (it is also the residual gradient of an identity block), and the reduction sums
// sum g and sum g (x - mean) are taken from the staged tile in bn_bwd_reduce_kernel's row plan (bn_bwd_reduce_plan:
// chunks of 128 rows, so whole tiles), thread layout and fp32 order, finished by its own code: bit-identical dbeta /
// dgamma.  Only moco_bn_bwd_apply_given is left to run.  The epilogue operands are x, dy2 and the mask bytes of the
// tile's 128 columns (66 KB per tile against 16-64 KB of mainloop operands); g is staged in place over dy2 and stored
// from there.
#include <cuda.h>
#include <cuda_bf16.h>

#include "../../include/moco_b200.h"
#include "bn_reduce.cuh"
#include "common.cuh"
#include "conv1x1_skeleton.cuh"
#include "sm90_ptx.cuh"
#include "tc_common.cuh"

namespace moco {

constexpr int kCvMaxSlabs = 64;            // 64-channel slabs (one ticket counter each in the workspace's 256 bytes)
constexpr int kCvMaxPartials = 528;        // workspace sizing: slabs x CTAs per slab of the statistics plan
static_assert(kBnStatsUnroll * kBnRows % kCvBM == 0, "a statistics chunk must be whole tiles");
static_assert(kBnThreads == 256, "the consumer warpgroups are the statistics pass's threads");

struct Conv1x1Args {
    int M, Cin, m_tiles, ppc, R, stages;   // ppc = tiles per CTA; R = CTAs per column slice
    int store;                             // 0: the statistics only, y is not written
    float momentum, eps;
    float* partial;                        // [slabs][R][128], bn_stats_kernel's layout
    unsigned int* counters;                // [slabs]
    float* mean;
    float* invstd;
    float* running_mean;                   // nullable (with running_var)
    float* running_var;
    long long* num_batches_tracked;        // nullable
};

// The epilogue operands' two buffers of kBytes: the producer loads those of tile iteration it into buffer it & 1, one
// tile ahead of the consumers, who hand the buffer back once the TMA store of the tile staged in it has read it.
template <int kBytes>
struct EpiRing {
    uint8_t* buf;                                                  // [2][kBytes]
    uint64_t* bar;                                                 // [2] full, [2] empty
    __device__ __forceinline__ uint8_t* tile(int it) const { return buf + (it & 1) * kBytes; }
    __device__ __forceinline__ uint64_t* full(int it) const { return &bar[it & 1]; }
    __device__ __forceinline__ uint64_t* empty(int it) const { return &bar[2 + (it & 1)]; }
    static __device__ __forceinline__ uint32_t parity(int it) { return (it >> 1) & 1; }
    __device__ __forceinline__ void init() const {
        for (int b = 0; b < 2; ++b) { mbar_init(full(b), 1); mbar_init(empty(b), kBnThreads); }
    }
    __device__ __forceinline__ void acquire(int it) const {      // producer, before its loads on full(it)
        mbar_wait(empty(it), parity(it) ^ 1u);
        mbar_arrive_expect_tx(full(it), (uint32_t)kBytes);        // OOB rows count too (zero-filled)
    }
    __device__ __forceinline__ void wait(int it) const { mbar_wait(full(it), parity(it)); }
    __device__ __forceinline__ void release(int it) const {      // every consumer thread
        if (threadIdx.x == 0) bulk_wait_read<0>();               // the store has read the tile out of the buffer
        mbar_arrive(empty(it));
    }
};

// The BatchNorm kernel's partials and finish, slab by slab, from sacc[s] (8 channels x 2 sums per consumer thread):
// in the last CTA of slab s to arrive, threads j < kBnSlab call finish(j, s, c) for channel j of the slab, channel c
// of the layer, with the slab totals in tot.
template <int kSlabs, typename Finish>
__device__ __forceinline__ void conv1x1_slabs_finish(float (&sacc)[kSlabs][16], float* red, double* tot, int* last,
                                                     float* partial, unsigned int* counters, int nb, int r, int R,
                                                     Finish finish) {
#pragma unroll
    for (int s = 0; s < kSlabs; ++s) {
        const int gs = nb * kSlabs + s;
        const float part = slab_reduce<2>(sacc[s], red, ConsumerSync());
        if (slab_finish<2>(part, partial, counters + gs, gs, r, R, tot, last, ConsumerSync()) && threadIdx.x < kBnSlab)
            finish((int)threadIdx.x, s, gs * kBnSlab + (int)threadIdx.x);
        consumer_sync();                                          // red / tot are reused by the next slab
    }
}

template <int BN>
__global__ void __launch_bounds__(kCvThreads, 1)
conv1x1_stats_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                     const __grid_constant__ CUtensorMap tm_y, const Conv1x1Args a) {
    using S = Conv1x1Shape<BN>;
    constexpr int kSlabs = BN / kBnSlab;
    extern __shared__ __align__(1024) uint8_t smem[];
    if ((smem_u32(smem) & 1023u) != 0u) __trap();
    const int NS = a.stages;
    uint8_t* ring = smem;                                          // NS x (x slab, w slab)
    uint8_t* outb = ring + (size_t)NS * S::kStage;                 // [buffer][warpgroup] output tiles
    float* shift_s = reinterpret_cast<float*>(outb + 4 * S::kOut); // [BN] y[0, c]
    float* red = shift_s + BN;                                     // [8 warps][kP]
    double* tot = reinterpret_cast<double*>(red + 8 * S::kP);      // [8 warps][kP]
    uint64_t* full = reinterpret_cast<uint64_t*>(tot + 8 * S::kP);
    uint64_t* empty = full + NS;
    int* last = reinterpret_cast<int*>(empty + NS);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nb = blockIdx.x, r = blockIdx.y;
    const int t0 = r * a.ppc;
    const int t1 = min(t0 + a.ppc, a.m_tiles);
    const int first = t0 > 0 ? -1 : 0;                             // iteration -1: tile 0 again, for the shift
    const int ksteps = a.Cin >> 6;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm_x);
        tma_prefetch_desc(&tm_w);
        tma_prefetch_desc(&tm_y);
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
            for (int it = first; it < t1 - t0; ++it)
                conv1x1_load_tile<BN, false>(&tm_x, &tm_w, ring, full, empty, NS, st, ph, it < 0 ? 0 : t0 + it, nb,
                                              ksteps);
        }
        return;
    }
    // ------------------------------------------------------------ consumer warpgroups
    setmaxnreg_inc<232>();
    const int wg = warp >> 2, t = threadIdx.x & 127;
    const int rloc = (warp & 3) * 16 + (lane >> 2);               // rows rloc and rloc + 8 of the warpgroup's 64
    const int ccol = 2 * (lane & 3);                              // first of this thread's two columns per 8
    const int v = threadIdx.x & (kBnLanes - 1), rl = threadIdx.x >> 3;   // bn_stats_kernel's thread layout
    float acc[BN / 2];
    float sacc[kSlabs][16];                                       // per slab: 8 sums of (y - h), 8 of (y - h)^2
    float sh[kSlabs][8];
#pragma unroll
    for (int s = 0; s < kSlabs; ++s)
#pragma unroll
        for (int k = 0; k < 16; ++k) sacc[s][k] = 0.f;
    int st = 0;
    uint32_t ph = 0;
    for (int it = first; it < t1 - t0; ++it) {
        const int tile = it < 0 ? 0 : t0 + it;
        conv1x1_mma_tile<BN, false>(acc, ring, wg, full, empty, NS, st, ph, ksteps, t);

        if (it == first) {                                        // tile 0: the shift y[0, c], as rounded
            if (wg == 0 && warp == 0 && lane < 4) {
#pragma unroll
                for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e)
                        shift_s[8 * j + ccol + e] = __bfloat162float(__float2bfloat16_rn(acc[4 * j + e]));
            }
            consumer_sync();
#pragma unroll
            for (int s = 0; s < kSlabs; ++s)
#pragma unroll
                for (int k = 0; k < 8; ++k) sh[s][k] = shift_s[s * kBnSlab + v * 8 + k];
            if (it < 0) continue;
        }

        // ---- epilogue: bf16 tile -> smem -> TMA store, and the statistics read back from the staged tile
        uint8_t* buf = outb + (it & 1) * 2 * S::kOut;             // [warpgroup] halves of this tile
        uint8_t* ob = buf + wg * S::kOut;
        if (t == 0) bulk_wait_read<1>();                          // the store that last used this buffer has read it
        warpgroup_sync(wg);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = rloc + 8 * h;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const __nv_bfloat162 q = __floats2bfloat162_rn(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                uint8_t* p = ob + (j >> 3) * 8192 + sw128_offset(row, j & 7) + (lane & 3) * 4;
                *reinterpret_cast<__nv_bfloat162*>(p) = q;
            }
        }
        fence_proxy_async();                                      // generic smem writes -> visible to the TMA store
        consumer_sync();                                 // both halves staged (and the buffer's last readers done)
        if (t == 0 && a.store) {
#pragma unroll
            for (int sl = 0; sl < BN / 64; ++sl)
                tma_store_2d(&tm_y, ob + sl * 8192, nb * BN + sl * 64, tile * kCvBM + wg * 64);
            bulk_commit();
        }
#pragma unroll
        for (int p = 0; p < kCvBM / kBnRows; ++p) {
            const int row = p * kBnRows + rl;
            if (tile * kCvBM + row < a.M) {
                const uint8_t* src = buf + (row >> 6) * S::kOut + sw128_offset(row & 63, v);
#pragma unroll
                for (int s = 0; s < kSlabs; ++s) {
                    float f[8];
                    unpack8(*reinterpret_cast<const uint4*>(src + s * 8192), f);
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        const float d = f[k] - sh[s][k];
                        sacc[s][k] += d;
                        sacc[s][8 + k] = fmaf(d, d, sacc[s][8 + k]);
                    }
                }
            }
        }
    }
    if (t == 0) bulk_wait<0>();

    conv1x1_slabs_finish(sacc, red, tot, last, a.partial, a.counters, nb, r, a.R, [&](int j, int s, int c) {
        bn_stats_channel(tot, j, shift_s[s * kBnSlab + j], a.M, a.eps, a.momentum, c, a.mean, a.invstd, a.running_mean,
                         a.running_var);
        if (c == 0 && a.num_batches_tracked != nullptr) *a.num_batches_tracked += 1;
    });
}

size_t conv1x1_workspace_bytes() { return 256 + (size_t)kCvMaxPartials * 2 * kBnSlab * sizeof(float); }

// The CTAs' row chunks of a BatchNorm pass's plan (bn_stats_plan, bn_bwd_reduce_plan), in 128-row tiles per CTA
static int tiles_per_cta(void (*plan)(long long, int, long long*, long long*, int*), long long M, int C, int* R) {
    long long passes = 0, ppc = 0;
    plan(M, C, &passes, &ppc, R);
    return (int)(ppc * kBnRows / kCvBM);
}

template <int BN>
static cudaError_t launch_stats(const void* x, const void* w, void* y, int M, int Cin, int Cout, const BnLayer& bn,
                                void* ws, cudaStream_t stream) {
    using S = Conv1x1Shape<BN>;
    Conv1x1Args a{};
    a.M = M; a.Cin = Cin;
    a.m_tiles = (M + kCvBM - 1) / kCvBM;
    a.ppc = tiles_per_cta(bn_stats_plan, M, Cout, &a.R);   // the statistics pass's row chunks
    const int slices = Cout / BN, slabs = Cout / kBnSlab;
    if (slabs > kCvMaxSlabs || (long long)slabs * a.R > kCvMaxPartials) return cudaErrorNotSupported;
    int smem = 0;
    const cudaError_t e = ring_smem(S::kFixed, S::kStage, &a.stages, &smem);
    if (e != cudaSuccess) return e;
    a.momentum = bn.momentum; a.eps = bn.eps;
    a.counters = static_cast<unsigned int*>(ws);
    a.partial = bn_ws_partials(ws);
    a.mean = bn.save_mean; a.invstd = bn.save_invstd;
    a.running_mean = bn.running_mean; a.running_var = bn.running_var; a.num_batches_tracked = bn.num_batches_tracked;
    a.store = y != nullptr;
    CUtensorMap tm_x, tm_w, tm_y;
    if (!make_tmap(&tm_x, x, M, Cin, kCvBM) || !make_tmap(&tm_w, w, Cout, Cin, BN))
        return cudaErrorUnknown;
    if (y == nullptr) tm_y = tm_x;                         // not used
    else if (!make_tmap(&tm_y, y, M, Cout, 64)) return cudaErrorUnknown;
    return launch_conv1x1<conv1x1_stats_kernel<BN>>(dim3(slices, a.R), smem, stream, tm_x, tm_w, tm_y, a);
}

bool conv1x1_stats_shape_ok(long long M, int Cin, int Cout) {
    return M >= 1 && M <= 0x7fffff80LL && Cin >= 64 && Cin % 64 == 0 && Cin <= 65536 && Cout >= 64 && Cout % 64 == 0 &&
           Cout <= 4096;
}

cudaError_t launch_conv1x1_bn_stats(const void* x, const void* w, void* y, long long M, int Cin, int Cout,
                                    const BnLayer& bn, void* ws, cudaStream_t stream) {
    if (!conv1x1_stats_shape_ok(M, Cin, Cout)) return cudaErrorNotSupported;
    if (Cout % 128 == 0) return launch_stats<128>(x, w, y, (int)M, Cin, Cout, bn, ws, stream);
    return launch_stats<64>(x, w, y, (int)M, Cin, Cout, bn, ws, stream);
}

// ---- the residual BatchNorm applied in a second pass of the GEMM ----------------------------------------------------
struct Conv1x1ApplyArgs {
    int M, Cin, C, m_tiles, ppc, stages;   // C = Cout; ppc = tiles per CTA
    const float* mean;
    const float* invstd;
    const float* gamma;
    const float* beta;
    const float* mean2;                    // kShortcut: the shortcut BN
    const float* invstd2;
    const float* gamma2;
    const float* beta2;
    uint8_t* mask;                         // nullable: uint8 [M, C / 8]
};

template <int BN>
struct Conv1x1ApplyShape {
    static constexpr int kTile = (BN / 64) * kSlab;        // r / y tile: [BN / 64 column slabs][128 rows x 64 bf16]
    static constexpr int kFixed = 2 * kTile + 4 * BN * 4;  // two tile buffers, ca / cb / ca2 / cb2
};

template <int BN, bool kShortcut>
__global__ void __launch_bounds__(kCvThreads, 1)
conv1x1_bn_apply_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                        const __grid_constant__ CUtensorMap tm_r, const __grid_constant__ CUtensorMap tm_y,
                        const Conv1x1ApplyArgs a) {
    using S = Conv1x1Shape<BN>;
    using E = Conv1x1ApplyShape<BN>;
    constexpr int kSlabs = BN / 64;
    extern __shared__ __align__(1024) uint8_t smem[];
    if ((smem_u32(smem) & 1023u) != 0u) __trap();
    const int NS = a.stages;
    uint8_t* ring = smem;                                          // NS x (x slab, w slab)
    uint8_t* epi = ring + (size_t)NS * S::kStage;
    float* ca = reinterpret_cast<float*>(epi + 2 * E::kTile);      // [BN] each
    float* cb = ca + BN;
    float* ca2 = cb + BN;
    float* cb2 = ca2 + BN;
    uint64_t* full = reinterpret_cast<uint64_t*>(cb2 + BN);
    uint64_t* empty = full + NS;
    const EpiRing<E::kTile> er{epi, empty + NS};                   // [2] r tiles, then y

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nb = blockIdx.x;
    const int t0 = blockIdx.y * a.ppc;
    const int t1 = min(t0 + a.ppc, a.m_tiles);
    const int ksteps = a.Cin >> 6;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm_x);
        tma_prefetch_desc(&tm_w);
        tma_prefetch_desc(&tm_r);
        tma_prefetch_desc(&tm_y);
        for (int s = 0; s < NS; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
        er.init();
        fence_mbar_init();
    }
    if (threadIdx.x < BN) {                                        // bn_apply_kernel's coefficients
        const int c = nb * BN + threadIdx.x;
        const float k = __ldg(a.gamma + c) * __ldg(a.invstd + c);
        ca[threadIdx.x] = k;
        cb[threadIdx.x] = fmaf(-__ldg(a.mean + c), k, __ldg(a.beta + c));
        if constexpr (kShortcut) {
            const float k2 = __ldg(a.gamma2 + c) * __ldg(a.invstd2 + c);
            ca2[threadIdx.x] = k2;
            cb2[threadIdx.x] = fmaf(-__ldg(a.mean2 + c), k2, __ldg(a.beta2 + c));
        }
    }
    __syncthreads();

    if (warp >= 8) {
        setmaxnreg_dec<40>();
        if (warp == 8 && elect_one()) {
            // ---------------------------------------------------- TMA producer
            int st = 0;
            uint32_t ph = 0;
            for (int it = 0; it < t1 - t0; ++it) {
                const int tile = t0 + it;
                er.acquire(it);
#pragma unroll
                for (int s = 0; s < kSlabs; ++s)
                    tma_load_2d(&tm_r, er.full(it), er.tile(it) + s * kSlab, nb * BN + s * 64, tile * kCvBM);
                conv1x1_load_tile<BN, false>(&tm_x, &tm_w, ring, full, empty, NS, st, ph, tile, nb, ksteps);
            }
        }
        return;
    }
    // ------------------------------------------------------------ consumer warpgroups
    setmaxnreg_inc<232>();
    const int wg = warp >> 2, t = threadIdx.x & 127;
    const int rloc = wg * 64 + (warp & 3) * 16 + (lane >> 2);    // tile rows rloc and rloc + 8
    const int ccol = 2 * (lane & 3);                              // first of this thread's two columns per 8
    const int v = threadIdx.x & (kBnLanes - 1), rl = threadIdx.x >> 3;   // 8-channel vector, row of the mask pass
    const int mask_row = a.C >> 3;
    float acc[BN / 2];
    int st = 0;
    uint32_t ph = 0;
    for (int it = 0; it < t1 - t0; ++it) {
        const int tile = t0 + it;
        conv1x1_mma_tile<BN, false>(acc, ring, wg, full, empty, NS, st, ph, ksteps, t);

        // ---- epilogue: y = relu(fmaf(bf16(acc), ca, cb) + r), in place over r -> TMA store; mask bytes from the tile
        uint8_t* e = er.tile(it);
        er.wait(it);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = rloc + 8 * h;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                __nv_bfloat162* p = reinterpret_cast<__nv_bfloat162*>(e + (j >> 3) * kSlab + sw128_offset(row, j & 7) +
                                                                      (lane & 3) * 4);
                const float2 r2 = __bfloat1622float2(*p);
                float z[2];
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const int c = 8 * j + ccol + q;
                    float r = q ? r2.y : r2.x;
                    if constexpr (kShortcut)
                        r = __bfloat162float(__float2bfloat16_rn(__fadd_rn(fmaf(r, ca2[c], cb2[c]), 0.f)));
                    const float hv = __bfloat162float(__float2bfloat16_rn(acc[4 * j + 2 * h + q]));
                    z[q] = fmaxf(__fadd_rn(fmaf(hv, ca[c], cb[c]), r), 0.f);
                }
                *p = __floats2bfloat162_rn(z[0], z[1]);
            }
        }
        fence_proxy_async();                                      // generic smem writes -> visible to the TMA store
        consumer_sync();                                          // the whole tile staged
        if (threadIdx.x == 0) {
#pragma unroll
            for (int s = 0; s < kSlabs; ++s) tma_store_2d(&tm_y, e + s * kSlab, nb * BN + s * 64, tile * kCvBM);
            bulk_commit();
        }
        if (a.mask != nullptr) {
#pragma unroll
            for (int p = 0; p < kCvBM / kBnRows; ++p) {
                const int row = p * kBnRows + rl;
                const long long grow = (long long)tile * kCvBM + row;
                if (grow < a.M) {
#pragma unroll
                    for (int s = 0; s < kSlabs; ++s) {
                        const uint4 u = *reinterpret_cast<const uint4*>(e + s * kSlab + sw128_offset(row, v));
                        a.mask[grow * mask_row + nb * (BN / 8) + s * 8 + v] = (uint8_t)relu_bits(u);
                    }
                }
            }
        }
        er.release(it);
    }
    if (threadIdx.x == 0) bulk_wait<0>();
}

template <int BN, bool SC>
static cudaError_t launch_apply(const void* x, const void* w, const void* res, void* y, void* mask, int M, int Cin,
                                int Cout, const BnLayer& bn, const BnLayer* sc, cudaStream_t stream) {
    using S = Conv1x1Shape<BN>;
    using E = Conv1x1ApplyShape<BN>;
    Conv1x1ApplyArgs a{};
    a.M = M; a.Cin = Cin; a.C = Cout;
    a.m_tiles = (M + kCvBM - 1) / kCvBM;
    int dev = 0, sms = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return e;
    const int slices = Cout / BN;
    int R = sms / slices;                                  // one CTA per SM
    if (R < 1) R = 1;
    a.ppc = (a.m_tiles + R - 1) / R;
    R = (a.m_tiles + a.ppc - 1) / a.ppc;
    int smem = 0;
    e = ring_smem(E::kFixed, S::kStage, &a.stages, &smem);
    if (e != cudaSuccess) return e;
    a.mean = bn.save_mean; a.invstd = bn.save_invstd; a.gamma = bn.gamma; a.beta = bn.beta;
    if (SC) { a.mean2 = sc->save_mean; a.invstd2 = sc->save_invstd; a.gamma2 = sc->gamma; a.beta2 = sc->beta; }
    a.mask = static_cast<uint8_t*>(mask);
    CUtensorMap tm_x, tm_w, tm_r, tm_y;
    if (!make_tmap(&tm_x, x, M, Cin, kCvBM) || !make_tmap(&tm_w, w, Cout, Cin, BN) ||
        !make_tmap(&tm_r, res, M, Cout, kCvBM) || !make_tmap(&tm_y, y, M, Cout, kCvBM))
        return cudaErrorUnknown;
    return launch_conv1x1<conv1x1_bn_apply_kernel<BN, SC>>(dim3(slices, R), smem, stream, tm_x, tm_w, tm_r, tm_y, a);
}

// Cout is the BatchNorm's C (a power of two in [64, 2048]), as in the statistics and apply passes it replaces
bool conv1x1_apply_shape_ok(long long M, int Cin, int Cout) {
    return M >= 1 && M <= 0x7fffff80LL && Cin >= 64 && Cin % 64 == 0 && Cin <= 65536 && Cout >= 64 && Cout <= 2048 &&
           (Cout & (Cout - 1)) == 0;
}

cudaError_t launch_conv1x1_bn_add_relu(const void* x, const void* w, const void* res, void* y, void* mask, long long M,
                                       int Cin, int Cout, const BnLayer& bn, const BnLayer* sc, int given, void* ws,
                                       cudaStream_t stream) {
    if (!conv1x1_apply_shape_ok(M, Cin, Cout)) return cudaErrorNotSupported;
    const int BN = Cout % 128 == 0 ? 128 : 64;
    cudaError_t e = cudaSuccess;
    if (!(given & MOCO_BN_STATS_GIVEN))                    // the statistics pass without storing h
        e = BN == 128 ? launch_stats<128>(x, w, nullptr, (int)M, Cin, Cout, bn, ws, stream)
                      : launch_stats<64>(x, w, nullptr, (int)M, Cin, Cout, bn, ws, stream);
    if (e == cudaSuccess && sc != nullptr && !(given & MOCO_BN_SC_STATS_GIVEN))
        e = launch_bn_stats(res, M, Cout, *sc, ws, stream);
    if (e != cudaSuccess) return e;
    if (BN == 128)
        return sc != nullptr ? launch_apply<128, true>(x, w, res, y, mask, (int)M, Cin, Cout, bn, sc, stream)
                             : launch_apply<128, false>(x, w, res, y, mask, (int)M, Cin, Cout, bn, sc, stream);
    return sc != nullptr ? launch_apply<64, true>(x, w, res, y, mask, (int)M, Cin, Cout, bn, sc, stream)
                         : launch_apply<64, false>(x, w, res, y, mask, (int)M, Cin, Cout, bn, sc, stream);
}

// ---- backward: the input gradient with the producing BatchNorm's backward reduction ---------------------------------
constexpr int kDgBN = 128;                       // columns of dX per CTA
struct DgradShape {                              // the epilogue's; the mainloop's are Conv1x1Shape<kDgBN>'s
    static constexpr int kTile = 2 * kSlab;              // [2 column slabs][128 rows x 64 bf16], 128-byte swizzle
    static constexpr int kMask = kCvBM * kDgBN / 8;      // [128 rows][16 mask bytes]
    static constexpr int kEpi = 2 * kTile + kMask;       // x tile, dy2 tile (then g), mask bytes
    // the two epilogue buffers, slab_reduce scratch (float), slab_finish totals (double)
    static constexpr int kFixed = 2 * kEpi + 8 * Conv1x1Shape<kDgBN>::kP * (4 + 8);
};
static_assert(kBnBwdReduceUnroll * kBnRows % kCvBM == 0, "a reduction chunk must be whole tiles");
static_assert(DgradShape::kEpi % 1024 == 0, "epilogue buffers keep the 1024-byte alignment of the swizzled tiles");

struct DgradArgs {
    int M, K, m_tiles, ppc, R, stages;   // K = Cout; ppc = tiles per CTA; R = CTAs per column slice
    float* partial;                      // [slabs][R][128], bn_bwd_reduce_kernel's layout
    unsigned int* counters;              // [slabs]
    const float* mean;
    const float* invstd;
    float* dgamma;
    float* dbeta;
};

__global__ void __launch_bounds__(kCvThreads, 1)
conv1x1_dgrad_bn_bwd_kernel(const __grid_constant__ CUtensorMap tm_dh, const __grid_constant__ CUtensorMap tm_w,
                            const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_dy2,
                            const __grid_constant__ CUtensorMap tm_mask, const __grid_constant__ CUtensorMap tm_g,
                            const DgradArgs a) {
    using S = Conv1x1Shape<kDgBN>;
    using E = DgradShape;
    constexpr int kSlabs = kDgBN / kBnSlab;
    extern __shared__ __align__(1024) uint8_t smem[];
    if ((smem_u32(smem) & 1023u) != 0u) __trap();
    const int NS = a.stages;
    uint8_t* ring = smem;                                          // NS x (dH slab, w slab)
    uint8_t* epi = ring + (size_t)NS * S::kStage;
    float* red = reinterpret_cast<float*>(epi + 2 * E::kEpi);      // [8 warps][kP]
    double* tot = reinterpret_cast<double*>(red + 8 * S::kP);      // [8 warps][kP]
    uint64_t* full = reinterpret_cast<uint64_t*>(tot + 8 * S::kP);
    uint64_t* empty = full + NS;
    const EpiRing<E::kEpi> er{epi, empty + NS};                    // [2] x (x tile, dy2 / g tile, mask bytes)
    int* last = reinterpret_cast<int*>(er.bar + 4);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nb = blockIdx.x, r = blockIdx.y;
    const int t0 = r * a.ppc;
    const int t1 = min(t0 + a.ppc, a.m_tiles);
    const int ksteps = a.K >> 6;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tm_dh);
        tma_prefetch_desc(&tm_w);
        tma_prefetch_desc(&tm_x);
        tma_prefetch_desc(&tm_dy2);
        tma_prefetch_desc(&tm_mask);
        tma_prefetch_desc(&tm_g);
        for (int s = 0; s < NS; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
        er.init();
        fence_mbar_init();
    }
    __syncthreads();

    if (warp >= 8) {
        setmaxnreg_dec<40>();
        if (warp == 8 && elect_one()) {
            // ---------------------------------------------------- TMA producer
            int st = 0;
            uint32_t ph = 0;
            for (int it = 0; it < t1 - t0; ++it) {
                const int tile = t0 + it, row0 = tile * kCvBM;
                uint8_t* e = er.tile(it);
                er.acquire(it);
#pragma unroll
                for (int s = 0; s < kSlabs; ++s) {
                    tma_load_2d(&tm_x, er.full(it), e + s * kSlab, nb * kDgBN + s * 64, row0);
                    tma_load_2d(&tm_dy2, er.full(it), e + E::kTile + s * kSlab, nb * kDgBN + s * 64, row0);
                }
                tma_load_2d(&tm_mask, er.full(it), e + 2 * E::kTile, nb * (kDgBN / 8), row0);
                conv1x1_load_tile<kDgBN, true>(&tm_dh, &tm_w, ring, full, empty, NS, st, ph, tile, nb, ksteps);
            }
        }
        return;
    }
    // ------------------------------------------------------------ consumer warpgroups
    setmaxnreg_inc<232>();
    const int wg = warp >> 2, t = threadIdx.x & 127;
    const int rloc = wg * 64 + (warp & 3) * 16 + (lane >> 2);    // tile rows rloc and rloc + 8
    const int ccol = 2 * (lane & 3);                              // first of this thread's two columns per 8
    const int v = threadIdx.x & (kBnLanes - 1), rl = threadIdx.x >> 3;   // bn_bwd_reduce_kernel's thread layout
    float acc[kDgBN / 2];
    float sacc[kSlabs][16];                                       // per slab: 8 sums of g, 8 of g (x - mean)
    float mu[kSlabs][8];
#pragma unroll
    for (int s = 0; s < kSlabs; ++s)
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            mu[s][k] = __ldg(a.mean + nb * kDgBN + s * kBnSlab + v * 8 + k);
            sacc[s][k] = sacc[s][8 + k] = 0.f;
        }
    int st = 0;
    uint32_t ph = 0;
    for (int it = 0; it < t1 - t0; ++it) {
        const int tile = t0 + it;
        conv1x1_mma_tile<kDgBN, true>(acc, ring, wg, full, empty, NS, st, ph, ksteps, t);

        // ---- epilogue: g = mask . bf16(bf16(dX) + dy2), in place over dy2 -> TMA store; the sums from the staged tile
        uint8_t* e = er.tile(it);
        uint8_t* gt = e + E::kTile;
        const uint8_t* mt = e + 2 * E::kTile;
        er.wait(it);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = rloc + 8 * h;
#pragma unroll
            for (int j = 0; j < kDgBN / 8; ++j) {
                __nv_bfloat162* p = reinterpret_cast<__nv_bfloat162*>(gt + (j >> 3) * kSlab + sw128_offset(row, j & 7) +
                                                                      (lane & 3) * 4);
                const float2 d2 = __bfloat1622float2(*p);
                const unsigned int bits = (unsigned int)mt[row * (kDgBN / 8) + j] >> ccol;
                const float d0 = __bfloat162float(__float2bfloat16_rn(acc[4 * j + 2 * h]));
                const float d1 = __bfloat162float(__float2bfloat16_rn(acc[4 * j + 2 * h + 1]));
                const float g0 = __bfloat162float(__float2bfloat16_rn(__fadd_rn(d0, d2.x)));
                const float g1 = __bfloat162float(__float2bfloat16_rn(__fadd_rn(d1, d2.y)));
                *p = __floats2bfloat162_rn((bits & 1u) ? g0 : 0.f, (bits & 2u) ? g1 : 0.f);
            }
        }
        fence_proxy_async();                                      // generic smem writes -> visible to the TMA store
        consumer_sync();                                          // the whole tile staged
        if (threadIdx.x == 0) {
#pragma unroll
            for (int s = 0; s < kSlabs; ++s) tma_store_2d(&tm_g, gt + s * kSlab, nb * kDgBN + s * 64, tile * kCvBM);
            bulk_commit();
        }
#pragma unroll
        for (int p = 0; p < kCvBM / kBnRows; ++p) {
            const int row = p * kBnRows + rl;
            if (tile * kCvBM + row < a.M) {
                const int off = sw128_offset(row, v);
#pragma unroll
                for (int s = 0; s < kSlabs; ++s) {
                    float g[8], f[8];
                    unpack8(*reinterpret_cast<const uint4*>(gt + s * kSlab + off), g);
                    unpack8(*reinterpret_cast<const uint4*>(e + s * kSlab + off), f);
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        sacc[s][k] += g[k];
                        sacc[s][8 + k] = fmaf(g[k], f[k] - mu[s][k], sacc[s][8 + k]);
                    }
                }
            }
        }
        er.release(it);
    }
    if (threadIdx.x == 0) bulk_wait<0>();

    conv1x1_slabs_finish(sacc, red, tot, last, a.partial, a.counters, nb, r, a.R, [&](int j, int, int c) {
        bn_bwd_channel<2>(tot, j, c, a.invstd, a.dbeta, a.dgamma, nullptr, nullptr, nullptr);
    });
}

// Cin is the BatchNorm's C (a power of two in [128, 2048]); Cout the GEMM's K
bool conv1x1_dgrad_shape_ok(long long M, int Cin, int Cout) {
    return M >= 1 && M <= 0x7fffff80LL && Cin >= kDgBN && Cin <= 2048 && (Cin & (Cin - 1)) == 0 && Cout >= 64 &&
           Cout % 64 == 0 && Cout <= 4096;
}

cudaError_t launch_conv1x1_dgrad_bn_bwd(const void* dh, const void* w, void* g, long long M, int Cin, int Cout,
                                        const void* x, const void* mask, const void* dy2, const BnLayer& bn, void* ws,
                                        cudaStream_t stream) {
    if (!conv1x1_dgrad_shape_ok(M, Cin, Cout)) return cudaErrorNotSupported;
    DgradArgs a{};
    a.M = (int)M; a.K = Cout;
    a.m_tiles = (int)((M + kCvBM - 1) / kCvBM);
    a.ppc = tiles_per_cta(bn_bwd_reduce_plan, M, Cin, &a.R);   // bn_bwd_reduce_kernel's row chunks
    const int slices = Cin / kDgBN, slabs = Cin / kBnSlab;
    if ((long long)slabs * a.R > kCvMaxPartials) return cudaErrorNotSupported;
    int smem = 0;
    const cudaError_t e = ring_smem(DgradShape::kFixed, Conv1x1Shape<kDgBN>::kStage, &a.stages, &smem);
    if (e != cudaSuccess) return e;
    a.counters = static_cast<unsigned int*>(ws);
    a.partial = bn_ws_partials(ws);
    a.mean = bn.save_mean; a.invstd = bn.save_invstd; a.dgamma = bn.dgamma; a.dbeta = bn.dbeta;
    CUtensorMap tm_dh, tm_w, tm_x, tm_dy2, tm_mask, tm_g;
    if (!make_tmap(&tm_dh, dh, (int)M, Cout, kCvBM) || !make_tmap(&tm_w, w, Cout, Cin, 64) ||
        !make_tmap(&tm_x, x, (int)M, Cin, kCvBM) || !make_tmap(&tm_dy2, dy2, (int)M, Cin, kCvBM) ||
        !encode_tmap(&tm_mask, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, CU_TENSOR_MAP_SWIZZLE_NONE, mask, (int)M, Cin / 8,
                     kCvBM, 16) ||                         // the mask bytes: [128 rows x 16 bytes] boxes, not swizzled
        !make_tmap(&tm_g, g, (int)M, Cin, kCvBM))
        return cudaErrorUnknown;
    return launch_conv1x1<conv1x1_dgrad_bn_bwd_kernel>(dim3(slices, a.R), smem, stream, tm_dh, tm_w, tm_x, tm_dy2,
                                                       tm_mask, tm_g, a);
}

}  // namespace moco
