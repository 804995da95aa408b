// The warp-specialised wgmma GEMM skeleton of the 1x1-convolution kernels (conv1x1_sm90.cu), shared with the kNN
// similarity sweep (knn_sm90.cu): the CTA layout, the TMA producer / wgmma consumer mainloop over one 128-row tile, the
// consumers' named barriers, the ring's smem plan and the launcher.  See conv1x1_sm90.cu's header for the layout.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>

#include "bn_reduce.cuh"
#include "common.cuh"
#include "sm90_ptx.cuh"
#include "tc_common.cuh"

namespace moco {

constexpr int kCvThreads = 384;            // 2 consumer warpgroups + 1 producer warpgroup (one TMA thread)
constexpr int kCvBM = 128;                 // rows per tile

template <int BN>
struct Conv1x1Shape {
    static constexpr int kA = kCvBM * 128;                 // A slab [128 rows x 64 bf16]
    static constexpr int kB = BN * 128;                    // B slab [BN x 64 bf16], or BN / 64 boxes [64 x 64 bf16]
    static constexpr int kStage = kA + kB;
    static constexpr int kOut = 64 * BN * 2;               // one warpgroup's [64 x BN] bf16 output tile
    static constexpr int kP = 2 * kBnSlab;                 // floats of a slab partial: two sums per channel
    // the statistics kernel's output buffers, shift, slab_reduce scratch, slab_finish totals
    static constexpr int kFixed = 4 * kOut + BN * 4 + 8 * kP * 4 + 8 * kP * 8;
};

// The consumers' named barriers (id 0 is __syncthreads'): both warpgroups, and warpgroup wg alone.
__device__ __forceinline__ void consumer_sync() { named_bar_sync(3, kBnThreads); }
__device__ __forceinline__ void warpgroup_sync(int wg) { named_bar_sync(1 + wg, 128); }
struct ConsumerSync {
    __device__ __forceinline__ void operator()() const { consumer_sync(); }
};

// The mainloop, one 128-row tile of column slice nb.  Producer: the ksteps chunks of the A slab and the B slab into the
// ring.  B is K-major, one [BN x 64] box of w [N, K] as stored, or MN-major, BN / 64 boxes [64 x 64] of w [K, N] as
// stored.  Consumers: wgmma over them in increasing K.  (st, ph): the ring position, carried from tile to tile.
template <int BN, bool kBMnMajor>
__device__ __forceinline__ void conv1x1_load_tile(const CUtensorMap* tm_a, const CUtensorMap* tm_b, uint8_t* ring,
                                                  uint64_t* full, uint64_t* empty, int NS, int& st, uint32_t& ph,
                                                  int tile, int nb, int ksteps) {
    using S = Conv1x1Shape<BN>;
    for (int kc = 0; kc < ksteps; ++kc) {
        mbar_wait(&empty[st], ph ^ 1u);
        mbar_arrive_expect_tx(&full[st], (uint32_t)S::kStage);   // OOB rows count too (zero-filled)
        uint8_t* s = ring + (size_t)st * S::kStage;
        tma_load_2d(tm_a, &full[st], s, kc * 64, tile * kCvBM);
        if constexpr (kBMnMajor) {
#pragma unroll
            for (int h = 0; h < BN / 64; ++h)
                tma_load_2d(tm_b, &full[st], s + S::kA + h * 64 * 128, nb * BN + h * 64, kc * 64);
        } else {
            tma_load_2d(tm_b, &full[st], s + S::kA, kc * 64, nb * BN);
        }
        if (++st == NS) { st = 0; ph ^= 1u; }
    }
}

template <int BN, bool kBMnMajor>
__device__ __forceinline__ void conv1x1_mma_tile(float (&acc)[BN / 2], const uint8_t* ring, int wg, uint64_t* full,
                                                 uint64_t* empty, int NS, int& st, uint32_t& ph, int ksteps, int t) {
    using S = Conv1x1Shape<BN>;
    constexpr uint64_t kStageUnits = S::kStage >> 4;
    constexpr uint64_t kBStep = kBMnMajor ? 128 : 2;              // k16 of B in 16-byte units: 16 rows, or 32 bytes
    const uint64_t a_desc0 = make_sw128_desc(smem_u32(ring + wg * 64 * 128), 16, 1024);
    const uint64_t b_desc0 = make_sw128_desc(smem_u32(ring + S::kA), kBMnMajor ? 64 * 128 : 16, 1024);
    int prev = 0;
    for (int kc = 0; kc < ksteps; ++kc) {
        mbar_wait(&full[st], ph);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint64_t a = a_desc0 + st * kStageUnits + 2 * k, b = b_desc0 + st * kStageUnits + kBStep * k;
            if constexpr (kBMnMajor) wgmma_ss_tb<BN>(acc, a, b, (kc | k) != 0);
            else                     wgmma_ss<BN>(acc, a, b, (kc | k) != 0);
        }
        wgmma_commit();
        wgmma_wait<1>();                                          // the previous chunk's wgmmas have completed
        if (kc > 0 && t == 0) mbar_arrive(&empty[prev]);
        prev = st;
        if (++st == NS) { st = 0; ph ^= 1u; }
    }
    wgmma_wait<0>();
    reg_fence(acc);
    if (t == 0) mbar_arrive(&empty[prev]);
}

// The ring's stage count and the kernel's dynamic smem: `fixed` bytes besides the ring, 256 bytes of mbarriers, and as
// many stages of `stage` bytes as fit, at most 8.  With fewer than 2 the loads could not overlap the wgmmas.
static inline cudaError_t ring_smem(int fixed, int stage, int* stages, int* smem) {
    int n = (kSmemBudget - fixed - 256) / stage;
    if (n > 8) n = 8;
    if (n < 2) return cudaErrorNotSupported;
    *stages = n;
    *smem = n * stage + fixed + 256;
    return cudaSuccess;
}

// Kern on a grid of kCvThreads-thread CTAs, its max-dynamic-smem attribute set first if this device needs it raised
template <auto Kern, typename... Params>
static cudaError_t launch_conv1x1(dim3 grid, int smem, cudaStream_t stream, const Params&... params) {
    {
        std::lock_guard<std::mutex> lock(g_kernel_cache_mutex);
        const cudaError_t e = set_max_smem(Kern, kernel_cache<Kern>(), smem);
        if (e != cudaSuccess) return e;
    }
    Kern<<<grid, kCvThreads, smem, stream>>>(params...);
    return launched();
}

}  // namespace moco
