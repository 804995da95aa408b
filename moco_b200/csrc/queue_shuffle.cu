// FIFO queue enqueue (moco/NCE/Contrast.py:29-34), fp32->bf16 cast, and the
// ShuffleBN peer-memory row gather (moco/util.py:47-58,69-93) with its
// cross-GPU signal barrier.  All HBM/NVLink-bound byte movers: 16-byte vector
// accesses, bulk-async (TMA) copies for large rows, grids sized from the SM count.
#include "common.cuh"
#include "sm90_ptx.cuh"

namespace moco {

// ---------------------------------------------------------------------------
// enqueue: queue[(index + i) mod K] = k_all[i]; one thread per 8 elements.
// index_dev != nullptr: the ring position is read from that device int64 instead of `index`, and the last block to
// finish (counted in `done`, zero on entry and re-armed here) advances it to (index + n_all) mod K once every block
// has read it -- the same device-side ring as the fused tail kernel's, so a captured graph replays correctly.
// ---------------------------------------------------------------------------
__device__ __forceinline__ long long enqueue_ring(long long index, const long long* index_dev) {
    return index_dev ? *index_dev : index;
}

__device__ __forceinline__ void enqueue_advance(long long ring, int n_all, long long K, long long* index_dev,
                                                unsigned int* done) {
    if (index_dev == nullptr) return;
    __syncthreads();                                   // every thread of this block has read the ring position
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(done, 1u) == gridDim.x - 1) {
            *index_dev = (ring + n_all) % K;
            *done = 0u;
        }
    }
}

__global__ void enqueue_kernel(__nv_bfloat16* __restrict__ qb, float* __restrict__ qf,
                               const void* __restrict__ k_all, int k_dtype, int n_all, int C, long long K,
                               long long index, long long row0, long long nrows, long long* index_dev,
                               unsigned int* done) {
    pdl_launch_dependents();
    pdl_wait();                  // the kernels that read the pre-enqueue queue (this step's head) are complete
    index = enqueue_ring(index, index_dev);
    const int vec_per_row = C >> 3;
    const long long total = (long long)n_all * vec_per_row;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        int i = (int)(t / vec_per_row), v = (int)(t % vec_per_row);
        long long dst = (index + i) % K - row0;       // ring slot, relative to the rows this buffer holds
        if (dst < 0 || dst >= nrows) continue;
        float f[8];
        if (k_dtype == 0) {
            const float4* src = reinterpret_cast<const float4*>(static_cast<const float*>(k_all) + (size_t)i * C) + v * 2;
            float4 a = src[0], b = src[1];
            f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
        } else {
            uint4 u = *(reinterpret_cast<const uint4*>(static_cast<const __nv_bfloat16*>(k_all) + (size_t)i * C) + v);
            const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
            for (int e = 0; e < 4; ++e) { float2 x = __bfloat1622float2(h[e]); f[2 * e] = x.x; f[2 * e + 1] = x.y; }
        }
        uint4 packed;
        __nv_bfloat162* ph = reinterpret_cast<__nv_bfloat162*>(&packed);
#pragma unroll
        for (int e = 0; e < 4; ++e) ph[e] = __floats2bfloat162_rn(f[2 * e], f[2 * e + 1]);
        *(reinterpret_cast<uint4*>(qb + (size_t)dst * C) + v) = packed;
        if (qf) {
            float4* d = reinterpret_cast<float4*>(qf + (size_t)dst * C) + v * 2;
            d[0] = make_float4(f[0], f[1], f[2], f[3]);
            d[1] = make_float4(f[4], f[5], f[6], f[7]);
        }
    }
    enqueue_advance(index, n_all, K, index_dev, done);
}

// scalar variant for C % 8 != 0
__global__ void enqueue_scalar_kernel(__nv_bfloat16* __restrict__ qb, float* __restrict__ qf,
                                      const void* __restrict__ k_all, int k_dtype, int n_all, int C, long long K,
                                      long long index, long long row0, long long nrows, long long* index_dev,
                                      unsigned int* done) {
    pdl_launch_dependents();
    pdl_wait();
    index = enqueue_ring(index, index_dev);
    const long long total = (long long)n_all * C;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        int i = (int)(t / C), c = (int)(t % C);
        long long dst = (index + i) % K - row0;
        if (dst < 0 || dst >= nrows) continue;
        float f = k_dtype == 0 ? static_cast<const float*>(k_all)[t]
                               : __bfloat162float(static_cast<const __nv_bfloat16*>(k_all)[t]);
        qb[(size_t)dst * C + c] = __float2bfloat16_rn(f);
        if (qf) qf[(size_t)dst * C + c] = f;
    }
    enqueue_advance(index, n_all, K, index_dev, done);
}

cudaError_t launch_enqueue(__nv_bfloat16* queue_bf16, float* queue_f32, const void* k_all, int k_dtype, int n_all,
                           int C, int64_t K, int64_t index, int64_t row0, int64_t nrows, cudaStream_t stream,
                           long long* index_dev, unsigned int* done) {
    if (n_all == 0) return cudaSuccess;
    if (index_dev != nullptr && done == nullptr) return cudaErrorInvalidValue;
    if ((C & 7) == 0) {
        long long total = (long long)n_all * (C >> 3);
        int blocks = (int)((total + 255) / 256);
        if (blocks > 132 * 8) blocks = 132 * 8;
        return launch_pdl(enqueue_kernel, dim3(blocks), dim3(256), 0, stream, queue_bf16, queue_f32, k_all, k_dtype, n_all, C,
                          (long long)K, (long long)index, (long long)row0, (long long)nrows, index_dev, done);
    } else {
        long long total = (long long)n_all * C;
        int blocks = (int)((total + 255) / 256);
        if (blocks > 132 * 8) blocks = 132 * 8;
        return launch_pdl(enqueue_scalar_kernel, dim3(blocks), dim3(256), 0, stream, queue_bf16, queue_f32, k_all, k_dtype,
                          n_all, C, (long long)K, (long long)index, (long long)row0, (long long)nrows, index_dev, done);
    }
    return cudaGetLastError();
}

__global__ void f32_to_bf16_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, size_t n) {
    size_t stride = (size_t)gridDim.x * blockDim.x;
    size_t n4 = n >> 2;
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < n4; t += stride) {
        float4 a = reinterpret_cast<const float4*>(src)[t];
        __nv_bfloat162 lo = __floats2bfloat162_rn(a.x, a.y), hi = __floats2bfloat162_rn(a.z, a.w);
        uint2 u;
        u.x = *reinterpret_cast<uint32_t*>(&lo);
        u.y = *reinterpret_cast<uint32_t*>(&hi);
        reinterpret_cast<uint2*>(dst)[t] = u;
    }
    for (size_t t = (n4 << 2) + (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += stride)
        dst[t] = __float2bfloat16_rn(src[t]);
}

cudaError_t launch_f32_to_bf16(const float* src, __nv_bfloat16* dst, size_t n, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    size_t blocks = (n / 4 + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (blocks == 0) blocks = 1;
    f32_to_bf16_kernel<<<(int)blocks, 256, 0, stream>>>(src, dst, n);
    return launched();
}

// ---------------------------------------------------------------------------
// ShuffleBN gather.
// ---------------------------------------------------------------------------
constexpr int kMaxWorld = 16;
struct PeerTable { const char* base[kMaxWorld]; };

// Small rows (feature vectors): one warp per destination row, 16-byte lanes.  (Its cross-GPU synchronisation, when
// requested, happens in the launch wrapper below: see gather_small_sync_kernel.)
__global__ void gather_small_kernel(PeerTable peers, int rows_per_rank, const int64_t* __restrict__ src_rows,
                                    int n_rows, int vec_per_row, uint4* __restrict__ dst) {
    int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n_rows) return;
    int lane = threadIdx.x & 31;
    long long g = src_rows[row];
    const uint4* src = reinterpret_cast<const uint4*>(peers.base[g / rows_per_rank]) + (size_t)(g % rows_per_rank) * vec_per_row;
    uint4* d = dst + (size_t)row * vec_per_row;
    for (int v = lane; v < vec_per_row; v += 32) d[v] = src[v];
}

// ---- cross-GPU synchronisation folded into the gather kernels ------------------------------------------------
// Every rank owns a signal pad (one uint32 slot per writer rank, peer-mapped).  "Event" number `epoch`:
//   signal : slot[rank] of EVERY peer's pad := epoch (release, system scope) -- "my staging buffer is published";
//   wait   : all `world` slots of MY OWN pad >= epoch (acquire) -- "every peer's buffer is published".
// With epoch == 0 the kernels skip both (single GPU, or the caller synchronised some other way).
// The wait is bounded in TIME (%globaltimer): on expiry the thread records {code, peer, epoch, waited ms} in a pinned
// host word block the host can read afterwards (moco_p2p_last_timeout) and then traps -- a stalled peer (checkpoint on
// rank 0, dataloader skew, a debugger) gives a diagnosable error instead of an opaque launch failure or a hang.
struct PadTable { uint32_t* pad[kMaxWorld]; };
struct SyncArgs {
    PadTable pads;
    int world, rank;
    uint32_t epoch;                 // 0: no synchronisation
    unsigned long long timeout_ns;
    unsigned int* status_host;      // pinned, mapped: [0] code, [1] peer, [2] epoch, [3] waited ms
};

__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ void peer_signal(const SyncArgs& sa, int p) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(sa.pads.pad[p] + sa.rank), "r"(sa.epoch) : "memory");
}

__device__ __forceinline__ void peer_wait(const SyncArgs& sa, int p) {
    const uint32_t* mine = sa.pads.pad[sa.rank] + p;
    uint32_t v;
    const unsigned long long t0 = globaltimer_ns();
    unsigned int polls = 0;
    for (;;) {
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(mine) : "memory");
        if ((int32_t)(v - sa.epoch) >= 0) return;
        if ((++polls & 1023u) == 0u) {
            const unsigned long long waited = globaltimer_ns() - t0;
            if (waited > sa.timeout_ns) {
                if (sa.status_host) {
                    sa.status_host[1] = (unsigned int)p;
                    sa.status_host[2] = sa.epoch;
                    sa.status_host[3] = (unsigned int)(waited / 1000000ull);
                    __threadfence_system();
                    sa.status_host[0] = 1u;             // MOCO_P2P_TIMEOUT
                    __threadfence_system();
                }
                __trap();
            }
        }
    }
}

// Small rows with the synchronisation folded in: block 0 publishes the signal, every block waits for all peers.
__global__ void gather_small_sync_kernel(PeerTable peers, SyncArgs sa, int rows_per_rank,
                                         const int64_t* __restrict__ src_rows, int n_rows, int vec_per_row,
                                         uint4* __restrict__ dst) {
    if (blockIdx.x == 0 && (int)threadIdx.x < sa.world) { __threadfence_system(); peer_signal(sa, threadIdx.x); }
    if ((int)threadIdx.x < sa.world) peer_wait(sa, threadIdx.x);
    __syncthreads();
    int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n_rows) return;
    int lane = threadIdx.x & 31;
    long long g = src_rows[row];
    const uint4* src = reinterpret_cast<const uint4*>(peers.base[g / rows_per_rank]) + (size_t)(g % rows_per_rank) * vec_per_row;
    uint4* d = dst + (size_t)row * vec_per_row;
    for (int v = lane; v < vec_per_row; v += 32) d[v] = src[v];
}

// Stand-alone event (no data movement attached): signal all peers, wait for all peers.
__global__ void signal_barrier_kernel(SyncArgs sa) {
    const int p = threadIdx.x;
    if (p >= sa.world) return;
    __threadfence_system();
    peer_signal(sa, p);
    peer_wait(sa, p);
}

// Large rows (images): a persistent grid of CTAs walks (row, chunk) work items.  Each item is a kChunk-byte
// bulk-async copy peer HBM -> smem (cp.async.bulk, completes on an mbarrier) followed by a bulk store smem -> local
// HBM, issued by ONE elected thread per CTA: the copy engines move the bytes over NVLink while the SM's warps stay
// free for a concurrently running kernel.  kStages - 1 loads are always in flight; a stage is refilled as soon as
// the store that drained it has finished READING shared memory (cp.async.bulk.wait_group.read 1: everything but the
// newest store), not after all outstanding stores (round 1: wait_group.read 0 drained the pipe once per item).
// Block 0 publishes this rank's signal first; every CTA waits for all peers' signals before its first pull.
constexpr int kChunk = 32 * 1024;
constexpr int kStages = 6;

__global__ void __launch_bounds__(32)
gather_bulk_kernel(PeerTable peers, SyncArgs sa, int rows_per_rank, const int64_t* __restrict__ src_rows, int n_rows,
                   unsigned long long row_bytes, char* __restrict__ dst) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) uint64_t full[kStages];
    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) mbar_init(&full[s], 1);
        fence_mbar_init();
    }
    __syncwarp();
    if (sa.epoch != 0u) {
        if (blockIdx.x == 0 && (int)threadIdx.x < sa.world) { __threadfence_system(); peer_signal(sa, threadIdx.x); }
        if ((int)threadIdx.x < sa.world) peer_wait(sa, threadIdx.x);
        __syncwarp();
    }
    if (!elect_one()) return;
    const unsigned long long chunks_per_row = (row_bytes + kChunk - 1) / kChunk;
    const unsigned long long total = chunks_per_row * (unsigned long long)n_rows;
    const unsigned long long first = blockIdx.x, stride = gridDim.x;
    const unsigned long long mine = first < total ? (total - first + stride - 1) / stride : 0ull;     // items of this CTA
    auto item = [&](unsigned long long k, const char*& s, char*& d, uint32_t& bytes) {
        // chunk-major order: consecutive CTAs work on consecutive ROWS (rows of a shuffled batch live on different
        // peers), so at any moment the pulls are spread over all source GPUs instead of 132 CTAs draining one row
        const unsigned long long it = first + k * stride;
        const unsigned long long row = it % (unsigned long long)n_rows, ch = it / (unsigned long long)n_rows;
        const long long g = src_rows[row];
        const unsigned long long off = ch * kChunk;
        bytes = (uint32_t)min((unsigned long long)kChunk, row_bytes - off);
        s = peers.base[g / rows_per_rank] + (unsigned long long)(g % rows_per_rank) * row_bytes + off;
        d = dst + row * row_bytes + off;
    };
    auto load = [&](unsigned long long k) {
        const int st = (int)(k % kStages);
        const char* s; char* d; uint32_t bytes;
        item(k, s, d, bytes);
        mbar_arrive_expect_tx(&full[st], bytes);
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(smem_u32(smem + (size_t)st * kChunk)), "l"(s), "r"(bytes), "r"(smem_u32(&full[st])) : "memory");
    };
    for (unsigned long long k = 0; k < mine && k < (unsigned long long)(kStages - 1); ++k) load(k);
    for (unsigned long long k = 0; k < mine; ++k) {
        const int st = (int)(k % kStages);
        mbar_wait(&full[st], (uint32_t)((k / kStages) & 1ull));
        const char* s; char* d; uint32_t bytes;
        item(k, s, d, bytes);
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                     ::"l"(d), "r"(smem_u32(smem + (size_t)st * kChunk)), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        if (k + kStages - 1 < mine) {
            // the stage item k + kStages - 1 lands in was drained by store k - 1: all but the newest store (k) must have
            // finished reading shared memory
            asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
            load(k + kStages - 1);
        }
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// Large rows, plain 16-byte LDG/STG path (fallback / comparison for the bulk-async kernel).
// grid = (segments per row, rows); each thread keeps 4 independent 16-byte loads in flight.
__global__ void __launch_bounds__(256)
gather_ldg_kernel(PeerTable peers, int rows_per_rank, const int64_t* __restrict__ src_rows, int n_rows,
                  unsigned long long vec_per_row, uint4* __restrict__ dst) {
    int row = blockIdx.y;
    long long g = src_rows[row];
    const uint4* src = reinterpret_cast<const uint4*>(peers.base[g / rows_per_rank]) + (unsigned long long)(g % rows_per_rank) * vec_per_row;
    uint4* d = dst + (unsigned long long)row * vec_per_row;
    unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    unsigned long long v = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; v + 3 * stride < vec_per_row; v += 4 * stride) {
        uint4 a = src[v], b = src[v + stride], c = src[v + 2 * stride], e = src[v + 3 * stride];
        d[v] = a; d[v + stride] = b; d[v + 2 * stride] = c; d[v + 3 * stride] = e;
    }
    for (; v < vec_per_row; v += stride) d[v] = src[v];
}

static unsigned long long barrier_timeout_ns() {
    static long long v = -1;
    if (v < 0) {
        const char* e = getenv("MOCO_BARRIER_TIMEOUT_MS");
        long long ms = e ? atoll(e) : 0;
        if (ms <= 0) ms = 120000;                          // two minutes: far above any legitimate skew of a training step
        v = ms * 1000000ll;
    }
    return (unsigned long long)v;
}

// pinned, device-mapped status words for the timeout diagnosis (one block per process; see moco_p2p_last_timeout)
unsigned int* p2p_status_words() {
    static unsigned int* host = nullptr;
    if (!host) {
        void* p = nullptr;
        if (cudaHostAlloc(&p, 64, cudaHostAllocPortable | cudaHostAllocMapped) == cudaSuccess) {
            host = static_cast<unsigned int*>(p);
            for (int i = 0; i < 16; ++i) host[i] = 0u;
        }
    }
    return host;
}

static SyncArgs make_sync(void* const* pads_host, int world, int rank, uint32_t epoch) {
    SyncArgs sa;
    for (int i = 0; i < kMaxWorld; ++i) sa.pads.pad[i] = (pads_host && i < world) ? static_cast<uint32_t*>(pads_host[i]) : nullptr;
    sa.world = world; sa.rank = rank; sa.epoch = pads_host ? epoch : 0u;
    sa.timeout_ns = barrier_timeout_ns();
    sa.status_host = p2p_status_words();
    return sa;
}

// pads_host == nullptr or epoch == 0: plain gather (no cross-GPU synchronisation inside the kernel)
cudaError_t launch_gather(const void* const* peers_host, int world, int rows_per_rank, const int64_t* src_rows,
                          int n_rows, size_t row_bytes, void* dst, int flags, cudaStream_t stream,
                          void* const* pads_host, int rank, uint32_t epoch) {
    if (world > kMaxWorld) return cudaErrorInvalidValue;
    const SyncArgs sa = make_sync(pads_host, world, rank, epoch);
    if (n_rows == 0) {
        if (sa.epoch == 0u) return cudaSuccess;
        signal_barrier_kernel<<<1, 32, 0, stream>>>(sa);   // still a participant of the event
        return launched();
    }
    PeerTable t;
    for (int i = 0; i < kMaxWorld; ++i) t.base[i] = i < world ? static_cast<const char*>(peers_host[i]) : nullptr;
    // AUTO: bulk-async copies for rows up to ~400 KB (bf16 images; one thread per SM instead of 8 warps), the 16-byte
    // load/store kernel above that (fp32 images, 602 KB rows)
    const bool use_ldg = (flags & 1) || row_bytes > (size_t)400 * 1024;
    if (row_bytes >= (size_t)kChunk / 2 && use_ldg) {
        if (sa.epoch != 0u) {
            signal_barrier_kernel<<<1, 32, 0, stream>>>(sa);
            const cudaError_t e = launched();
            if (e != cudaSuccess) return e;
        }
        unsigned long long vec = row_bytes / 16;
        int gx = (int)((vec + 256 * 4 - 1) / (256 * 4));
        if (gx > 8) gx = 8;
        gather_ldg_kernel<<<dim3(gx, n_rows), 256, 0, stream>>>(t, rows_per_rank, src_rows, n_rows, vec,
                                                                static_cast<uint4*>(dst));
    } else if (row_bytes >= (size_t)kChunk / 2) {
        static bool attr_set[64] = {false};
        const int smem = kStages * kChunk;
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
        if (!attr_set[dev]) {
            cudaError_t e = cudaFuncSetAttribute(gather_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
            if (e != cudaSuccess) return e;
            attr_set[dev] = true;
        }
        size_t chunks = (row_bytes + kChunk - 1) / kChunk * (size_t)n_rows;
        int grid = (int)(chunks < 132 ? chunks : 132);
        gather_bulk_kernel<<<grid, 32, smem, stream>>>(t, sa, rows_per_rank, src_rows, n_rows, row_bytes,
                                                       static_cast<char*>(dst));
    } else {
        int vec = (int)(row_bytes / 16);
        int rows_per_block = 8;
        int blocks = (n_rows + rows_per_block - 1) / rows_per_block;
        if (sa.epoch != 0u)
            gather_small_sync_kernel<<<blocks, rows_per_block * 32, 0, stream>>>(t, sa, rows_per_rank, src_rows, n_rows, vec,
                                                                                static_cast<uint4*>(dst));
        else
            gather_small_kernel<<<blocks, rows_per_block * 32, 0, stream>>>(t, rows_per_rank, src_rows, n_rows, vec,
                                                                           static_cast<uint4*>(dst));
    }
    return launched();
}

cudaError_t launch_signal_barrier(void* const* pads_host, int world, int rank, uint32_t epoch, cudaStream_t stream) {
    if (world > kMaxWorld) return cudaErrorInvalidValue;
    signal_barrier_kernel<<<1, 32, 0, stream>>>(make_sync(pads_host, world, rank, epoch));
    return launched();
}

}  // namespace moco

// ---------------------------------------------------------------------------
// Input path: one crop of the NCHW batch -> bf16 NHWC (channels_last storage), one pass.
// Reference: train.py:250-254 splits the 6-channel batch into two crops; Apex/autocast then casts to half and
// cuDNN converts the layout in front of the first convolution (two more passes over the images).  Here the crop
// selection (strided read), the cast and the layout change are one kernel; its output is what the ShuffleBN
// gather publishes / pulls, so the key encoder's first conv reads exactly what crossed NVLink.
// Each thread converts 8 consecutive pixels: C plane reads of 32 B, one contiguous 16*C-byte store.
// ---------------------------------------------------------------------------
namespace moco {

template <int C, typename SrcT>
__global__ void __launch_bounds__(256)
crop_to_nhwc_kernel(const SrcT* __restrict__ src, long long img_stride, __nv_bfloat16* __restrict__ dst, int N, int HW,
                    const int64_t* __restrict__ src_rows) {
    pdl_launch_dependents();
    pdl_wait();
    const int groups = HW >> 3;                                   // 8-pixel groups per image
    const long long total = (long long)N * groups;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(t / groups), gidx = (int)(t % groups);
        // src_rows: output image n is input image src_rows[n] (single-GPU ShuffleBN: the permutation is the address)
        const SrcT* s = src + (size_t)(src_rows ? src_rows[n] : n) * img_stride + (size_t)gidx * 8;
        float v[C][8];
#pragma unroll
        for (int c = 0; c < C; ++c) {
            if constexpr (sizeof(SrcT) == 4) {
                const float4 a = *reinterpret_cast<const float4*>(s + (size_t)c * HW);
                const float4 b = *reinterpret_cast<const float4*>(s + (size_t)c * HW + 4);
                v[c][0] = a.x; v[c][1] = a.y; v[c][2] = a.z; v[c][3] = a.w;
                v[c][4] = b.x; v[c][5] = b.y; v[c][6] = b.z; v[c][7] = b.w;
            } else {
                const uint4 u = *reinterpret_cast<const uint4*>(s + (size_t)c * HW);
                const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
                for (int e = 0; e < 4; ++e) { float2 f = __bfloat1622float2(h[e]); v[c][2 * e] = f.x; v[c][2 * e + 1] = f.y; }
            }
        }
        // interleave: out[p * C + c]
        __align__(16) __nv_bfloat16 o[8 * C];
#pragma unroll
        for (int p = 0; p < 8; ++p)
#pragma unroll
            for (int c = 0; c < C; ++c) o[p * C + c] = __float2bfloat16_rn(v[c][p]);
        uint4* d = reinterpret_cast<uint4*>(dst + ((size_t)n * HW + (size_t)gidx * 8) * C);
#pragma unroll
        for (int w = 0; w < C; ++w) d[w] = reinterpret_cast<const uint4*>(o)[w];        // 8*C bf16 = C x 16 bytes
    }
}

// The same crop, written in the layout a space-to-depth stem reads: the reference's first convolution
// (moco/models/resnet.py:112, 7x7 / stride 2 / pad 3 on 3 channels) equals a 4x4 / stride 1 / pad 0 convolution over
//     s[n, R, Q, (b * 2 + d) * 3 + c] = x[n, c, 2 (R - 2) + b, 2 (Q - 2) + d]     (0 outside the image; channels 12..15 = 0)
// with R < H/2 + 3, Q < W/2 + 3 (two zero rows / columns in front, one behind: the 7-tap window padded to 8 taps),
// and 16 input channels are what cuDNN's implicit-GEMM kernels want (C = 3 runs a legacy kernel at 2 % of
// peak plus channel-padding passes).  One thread per output pixel: 6 coalesced 8-byte (fp32) or 4-byte (bf16) loads,
// two 16-byte stores.
template <typename SrcT>
__global__ void __launch_bounds__(256)
crop_to_s2d_kernel(const SrcT* __restrict__ src, long long img_stride, __nv_bfloat16* __restrict__ dst, int N, int H, int W,
                   const int64_t* __restrict__ src_rows) {
    pdl_launch_dependents();
    pdl_wait();
    const int R = (H >> 1) + 3, Q = (W >> 1) + 3;
    const long long total = (long long)N * R * Q;
    const size_t HW = (size_t)H * W;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int q = (int)(t % Q);
        const long long t2 = t / Q;
        const int r = (int)(t2 % R), n = (int)(t2 / R);
        __align__(16) __nv_bfloat16 o[16];
#pragma unroll
        for (int e = 0; e < 16; ++e) o[e] = __float2bfloat16_rn(0.f);
        const int h0 = 2 * (r - 2), w0 = 2 * (q - 2);
        if (h0 >= 0 && h0 < H && w0 >= 0 && w0 < W) {
            const SrcT* s = src + (size_t)(src_rows ? src_rows[n] : n) * img_stride + (size_t)h0 * W + w0;
#pragma unroll
            for (int b = 0; b < 2; ++b)
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    float v0, v1;
                    if constexpr (sizeof(SrcT) == 4) {
                        const float2 f = *reinterpret_cast<const float2*>(s + (size_t)c * HW + (size_t)b * W);
                        v0 = f.x; v1 = f.y;
                    } else {
                        const __nv_bfloat162 f = *reinterpret_cast<const __nv_bfloat162*>(s + (size_t)c * HW + (size_t)b * W);
                        v0 = __bfloat162float(f.x); v1 = __bfloat162float(f.y);
                    }
                    o[(b * 2 + 0) * 3 + c] = __float2bfloat16_rn(v0);
                    o[(b * 2 + 1) * 3 + c] = __float2bfloat16_rn(v1);
                }
        }
        uint4* d = reinterpret_cast<uint4*>(dst + (size_t)t * 16);
        d[0] = reinterpret_cast<const uint4*>(o)[0];
        d[1] = reinterpret_cast<const uint4*>(o)[1];
    }
}

cudaError_t launch_crop_to_s2d(const void* src, int src_dtype, long long img_stride, __nv_bfloat16* dst, int N, int H, int W,
                               cudaStream_t stream, const int64_t* src_rows) {
    if (N == 0) return cudaSuccess;
    if (H < 2 || W < 2 || (H & 1) || (W & 1)) return cudaErrorNotSupported;
    const long long total = (long long)N * ((H >> 1) + 3) * ((W >> 1) + 3);
    long long blocks = (total + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (src_dtype == 0)
        return launch_pdl(crop_to_s2d_kernel<float>, dim3((unsigned)blocks), dim3(256), 0, stream,
                          static_cast<const float*>(src), img_stride, dst, N, H, W, src_rows);
    return launch_pdl(crop_to_s2d_kernel<__nv_bfloat16>, dim3((unsigned)blocks), dim3(256), 0, stream,
                      static_cast<const __nv_bfloat16*>(src), img_stride, dst, N, H, W, src_rows);
}

cudaError_t launch_crop_to_nhwc(const void* src, int src_dtype, long long img_stride, __nv_bfloat16* dst, int N, int C,
                                int HW, cudaStream_t stream, const int64_t* src_rows) {
    if (N == 0) return cudaSuccess;
    if (C < 1 || C > 4 || (HW & 7) != 0) return cudaErrorNotSupported;
    const long long total = (long long)N * (HW >> 3);
    long long blocks = (total + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
#define MOCO_CROP(C_)                                                                                                 \
    if (C == C_) {                                                                                                    \
        if (src_dtype == 0)                                                                                           \
            return launch_pdl(crop_to_nhwc_kernel<C_, float>, dim3((unsigned)blocks), dim3(256), 0, stream,            \
                              static_cast<const float*>(src), img_stride, dst, N, HW, src_rows);                      \
        return launch_pdl(crop_to_nhwc_kernel<C_, __nv_bfloat16>, dim3((unsigned)blocks), dim3(256), 0, stream,        \
                          static_cast<const __nv_bfloat16*>(src), img_stride, dst, N, HW, src_rows);                  \
    }
    MOCO_CROP(1) MOCO_CROP(2) MOCO_CROP(3) MOCO_CROP(4)
#undef MOCO_CROP
    return cudaErrorNotSupported;
}

}  // namespace moco
