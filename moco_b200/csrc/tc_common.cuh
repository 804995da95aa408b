// Shared pieces of the tensor-core (wgmma) kernels' translation units: smem constants, tensor-map creation, and
// the persistent-grid launch planner (cluster-aware).
#pragma once
#include <cuda.h>
#include <stdlib.h>

#include <mutex>

#include "common.cuh"
#include "sm90_ptx.cuh"

namespace moco {

constexpr int kSlab = 128 * 128;            // bytes of a [128 rows x 64 bf16] swizzled slab
constexpr int kSmemBudget = 232448 - 1024;  // max dynamic smem per CTA on sm_90 (227 KB) minus alignment slack

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// Byte offset of 16-byte chunk `chunk` (8 bf16, < 8) of row `row` in a [rows x 64 bf16] slab in the 128-byte-swizzle
// layout of TMA and wgmma: rows of 128 bytes, chunk c of row r at position c ^ (r & 7).
__device__ __forceinline__ int sw128_offset(int row, int chunk) { return row * 128 + ((chunk ^ (row & 7)) << 4); }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn) return fn;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess || p == nullptr)
        return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(p);
    return fn;
}

// [rows, cols] row-major tensor of `elem`-byte elements, box = [box_rows, box_cols], OOB -> zeros.
inline bool encode_tmap(CUtensorMap* m, CUtensorMapDataType type, int elem, CUtensorMapSwizzle swizzle,
                        const void* base, int rows, int cols, int box_rows, int box_cols) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) { set_error("cuTensorMapEncodeTiled entry point not available"); return false; }
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)cols * elem};
    cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1u, 1u};
    CUresult r = fn(m, type, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (CUresult %d)", (int)r); return false; }
    return true;
}

// [rows, C] bf16 row-major tensor, box = [box_rows, 64 elements], 128B swizzle, OOB -> zeros.
inline bool make_tmap(CUtensorMap* m, const void* base, int rows, int C, int box_rows) {
    return encode_tmap(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, CU_TENSOR_MAP_SWIZZLE_128B, base, rows, C, box_rows, 64);
}

// Per-kernel launch state: the max-dynamic-smem attribute is set once, and the number of clusters that can be
// co-resident (persistent grid: one wave) is queried once per (smem, cluster) -- a cluster size > 1 can strand SMs
// in GPCs whose SM count is not a multiple of it, so it is NOT simply #SM / cluster.
struct KernelCache {
    int smem_set = -1;
    int q_smem = -1, q_cluster = -1, q_result = 0;
};

// cudaFuncSetAttribute and the occupancy answer are per DEVICE: one cache entry per (device ordinal, kernel), all
// guarded by one mutex (launches from several host threads / several GPUs in one process).
constexpr int kMaxDevices = 64;
static std::mutex g_kernel_cache_mutex;
template <auto Kern>
static KernelCache& kernel_cache() {
    static KernelCache table[kMaxDevices];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = 0;
    return table[dev];
}

// Raises the kernel's max-dynamic-smem attribute to smem unless an earlier launch on this device already did; called
// under g_kernel_cache_mutex.
template <typename Kern>
static cudaError_t set_max_smem(Kern kern, KernelCache& kc, int smem) {
    if (kc.smem_set >= smem) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e == cudaSuccess) kc.smem_set = smem;
    return e;
}

template <auto Kern>
static cudaError_t prepare_kernel(int threads, int smem, int cluster, int* max_clusters) {
    KernelCache& kc = kernel_cache<Kern>();
    const bool first = kc.smem_set < smem;
    cudaError_t e = set_max_smem(Kern, kc, smem);
    if (e != cudaSuccess) return e;
    if (first && cluster > 1) {
        e = cudaFuncSetAttribute(Kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 0);
        (void)e;
        cudaGetLastError();
    }
    if (kc.q_smem != smem || kc.q_cluster != cluster) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(cluster * 64);
        cfg.blockDim = dim3(threads);
        cfg.dynamicSmemBytes = smem;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = cluster;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        int n = 0;
        e = cudaOccupancyMaxActiveClusters(&n, Kern, &cfg);
        if (e != cudaSuccess) return e;
        kc.q_smem = smem; kc.q_cluster = cluster; kc.q_result = n;
    }
    *max_clusters = kc.q_result;
    return cudaSuccess;
}

template <typename Kern, typename Args>
static cudaError_t launch_cluster(Kern kern, int grid, int threads, int smem, int cluster, cudaStream_t stream,
                                  const CUtensorMap& tmap, const Args& args, bool pdl = false) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(threads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    int n = 0;
    if (cluster > 1) {                          // plain launch when no cluster feature is used
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = cluster;
        attr[n].val.clusterDim.y = 1;
        attr[n].val.clusterDim.z = 1;
        ++n;
    }
    if (pdl && pdl_enabled()) {                 // only for kernels that call pdl_wait() (common.cuh)
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    cfg.attrs = attr;
    cfg.numAttrs = n;
    return counted(cudaLaunchKernelEx(&cfg, kern, tmap, args));
}

// plan + launch one templated kernel instance: `fill(slices)` finalises the argument struct
template <auto Kern, typename Args, typename Fill>
static cudaError_t plan_and_launch(int threads, int smem, int cluster, int mgroups, int ctas_per_slice, int num_tiles,
                                   int n_pad, int* slices_out, cudaStream_t stream, const CUtensorMap& tmap, Args& args,
                                   Fill fill, bool pdl = false, bool plan_only = false) {
    int max_clusters = 0;
    cudaError_t e;
    {
        std::lock_guard<std::mutex> lock(g_kernel_cache_mutex);
        e = prepare_kernel<Kern>(threads, smem, cluster, &max_clusters);
    }
    if (e != cudaSuccess) return e;
    int slices = max_clusters / mgroups;            // one persistent wave
    if (slices > num_tiles) slices = num_tiles;
    if (slices < 1) return cudaErrorNotSupported;
    while ((size_t)slices * n_pad > (size_t)kMaxCtas * kRowsPerCta) --slices;
    if (slices < 1) return cudaErrorNotSupported;
    *slices_out = slices;
    if (plan_only) return cudaSuccess;          // the caller only needs the (deterministic) slice count
    fill(args, slices);
    return launch_cluster(Kern, ctas_per_slice * slices, threads, smem, cluster, stream, tmap, args, pdl);
}

}  // namespace moco
