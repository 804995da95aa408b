// extern "C" boundary of libmoco_b200.so (see include/moco_b200.h).
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include "../../include/moco_b200.h"
#include "common.cuh"

namespace moco {

static thread_local char g_err[512] = "";
std::atomic<unsigned long long> g_launch_count{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

struct DevInfo { int sms; int major; int minor; bool ok; };
static DevInfo device_info() {
    static DevInfo cache[64];
    static bool have[64] = {false};
    int dev = 0;
    DevInfo d = {0, 0, 0, false};
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return d;
    if (have[dev]) return cache[dev];
    if (cudaDeviceGetAttribute(&d.sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return d;
    cudaDeviceGetAttribute(&d.major, cudaDevAttrComputeCapabilityMajor, dev);
    cudaDeviceGetAttribute(&d.minor, cudaDevAttrComputeCapabilityMinor, dev);
    d.ok = true;
    cache[dev] = d;
    have[dev] = true;
    return d;
}

// optional profiling hook: CUDA events recorded right before / after one kernel of moco_nce_fwd
static cudaEvent_t g_prof_ev[3][2] = {{nullptr, nullptr}, {nullptr, nullptr}, {nullptr, nullptr}};
static inline void prof_mark(int kernel, int which, cudaStream_t s) {
    if (g_prof_ev[kernel][which]) cudaEventRecord(g_prof_ev[kernel][which], s);
}

// p is a multiple of `bytes` (a power of two) apart from NULL; NULL counts as aligned (the caller checks for NULL)
static bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }
// a required activation / workspace pointer: not NULL, and aligned for the kernels' 16-byte vectors
static bool ptr16(const void* p) { return p && aligned(p, 16); }

// An entry point's refusal of its arguments: "<fn>: <message>" for moco_last_error(), and `code` returned.
static int refuse(const char* fn, int code, const char* fmt, ...) {
    char msg[sizeof(g_err)];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(msg, sizeof(msg), fmt, ap);
    va_end(ap);
    set_error("%s: %s", fn, msg);
    return code;
}

// How an entry point ends once its CUDA work is issued: cudaSuccess is MOCO_OK.  cudaErrorNotSupported (a shape outside
// the launcher's envelope) is MOCO_ERR_UNSUPPORTED, worded by the printf-style `unsupported`, or generically after
// `what` when that is NULL.  Anything else is MOCO_ERR_CUDA after `what`, except that a cudaErrorUnknown keeps a
// message the launcher set (make_tmap sets one; every entry point clears g_err before its launches).
static int cuda_result(cudaError_t e, const char* what, const char* unsupported = nullptr, ...) {
    if (e == cudaSuccess) return MOCO_OK;
    if (e == cudaErrorNotSupported) {
        if (!unsupported) {
            set_error("%s: shape/device not supported by this kernel", what);
        } else {
            va_list ap;
            va_start(ap, unsupported);
            vsnprintf(g_err, sizeof(g_err), unsupported, ap);
            va_end(ap);
        }
        return MOCO_ERR_UNSUPPORTED;
    }
    if (g_err[0] == 0 || e != cudaErrorUnknown) set_error("%s: %s", what, cudaGetErrorString(e));
    return MOCO_ERR_CUDA;
}

// the wgmma kernels: an sm_90 device and a C they take
static bool tc_available(const DevInfo& d, int C) { return d.ok && d.major == 9 && nce_tc_shape_ok(C); }

// What every training BatchNorm entry point does once its arguments are checked: the workspace check (reduces: a
// statistics / reduction pass runs), then the launch of its plan.
template <typename Plan>
static int bn_launch(const char* fn, cudaError_t (*launch)(const Plan&, cudaStream_t), const Plan& plan, bool reduces,
                     size_t workspace_bytes, void* stream_) {
    if (reduces && workspace_bytes < bn_workspace_bytes()) return refuse(fn, MOCO_ERR_WORKSPACE, "workspace too small");
    return cuda_result(launch(plan, static_cast<cudaStream_t>(stream_)), fn, "%s: needs M >= 1 and C a power of two in "
                       "[64, 2048]; moco_bn_bwd_apply_given takes no shortcut BN (M=%lld C=%d)", fn, plan.M, plan.C);
}

}  // namespace moco

using namespace moco;

extern "C" {

int moco_abi_version(void) { return MOCO_B200_ABI_VERSION; }

const char* moco_last_error(void) { return g_err; }

int moco_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    DevInfo d = device_info();
    if (!d.ok) return refuse("moco_device_info", MOCO_ERR_CUDA, "no CUDA device");
    if (sm_count) *sm_count = d.sms;
    if (cc_major) *cc_major = d.major;
    if (cc_minor) *cc_minor = d.minor;
    return MOCO_OK;
}

unsigned long long moco_launch_count(void) { return g_launch_count.load(std::memory_order_relaxed); }

size_t moco_nce_workspace_bytes(int N, int C, int K) {
    (void)K;
    if (N <= 0 || C <= 0) return 0;
    return carve_workspace(nullptr, N, C).bytes;
}

}  // extern "C"

// The q.Queue^T sweep (one-sweep mode when lse == nullptr, nce_sweep_sm90.cu): C in {64, 128} reads q as given
// (fp32/bf16, optional L2 normalisation); C in {192, 256} reads the bf16 copy `qb` (a 16-byte piece of an fp32 row
// per thread would not keep a row inside one warp for the norm).
static cudaError_t launch_sweep(const void* q, int q_dtype, int normalize, const __nv_bfloat16* qb,
                                const __nv_bfloat16* queue, int N, int C, int K, float inv_T, const float* lse, int sms,
                                int* slices, int* n_pad, const NceWorkspace& ws, cudaStream_t stream,
                                bool plan_only = false) {
    if (C == 64 || C == 128)
        return launch_nce_sweep(q, q_dtype, normalize, queue, N, C, K, inv_T, lse, sms, slices, n_pad, ws, stream, plan_only);
    if (normalize) return cudaErrorNotSupported;
    return launch_nce_sweep(qb, MOCO_BF16, 0, queue, N, C, K, inv_T, lse, sms, slices, n_pad, ws, stream, plan_only);
}

// the statistics sweep on the wgmma kernels over `queue` (K rows); slices / n_pad are set by the launch
static NceTcParams tc_params(const __nv_bfloat16* qb, const void* queue, int N, int C, int K, float inv_T, float* logits,
                             int flags, int sms) {
    NceTcParams p;
    p.q_bf16 = qb; p.queue = static_cast<const __nv_bfloat16*>(queue); p.N = N; p.C = C; p.K = K; p.inv_T = inv_T;
    p.logits = logits;
    p.cta_group = (flags & MOCO_NCE_CTA_PAIR) ? 2 : 1;
    p.num_sms = sms;
    p.slices = 0; p.n_pad = 0;
    return p;
}

struct EnqueueSpec {            // n_all == 0: no enqueue
    void* queue_bf16; float* queue_f32; const void* k_all; int k_dtype; int n_all;
    long long index; long long* index_dev;
};

// the enqueue of moco_nce_step as a kernel of its own, on the paths whose last kernel does not do it
static int nce_enqueue(const EnqueueSpec& enq, int C, int K, const NceWorkspace& ws, cudaStream_t stream) {
    if (enq.n_all <= 0) return MOCO_OK;
    return cuda_result(launch_enqueue(static_cast<__nv_bfloat16*>(enq.queue_bf16), enq.queue_f32, enq.k_all, enq.k_dtype,
                                      enq.n_all, C, K, enq.index, 0, K, stream, enq.index_dev, ws.counters + 2),
                       "enqueue kernel");
}

static int nce_head(const void* q, const void* k, int qk_dtype, int normalize, const void* queue_bf16, int N, int C,
                    int K, float inv_T, float* logits, float* lse, float* loss_rows, float* prob_rows, float* loss_prob,
                    float* dq, void* workspace, size_t workspace_bytes, int flags, const EnqueueSpec& enq,
                    cudaStream_t stream, const char* who) {
    g_err[0] = 0;
    if (!q || !k || !queue_bf16 || !lse || !loss_rows || !prob_rows || !loss_prob || !workspace)
        return refuse(who, MOCO_ERR_INVALID, "null pointer argument");
    if (N <= 0 || C <= 0 || K <= 0 || !(inv_T > 0.f) || (qk_dtype != MOCO_F32 && qk_dtype != MOCO_BF16))
        return refuse(who, MOCO_ERR_INVALID, "bad N/C/K/inv_T/dtype (N=%d C=%d K=%d inv_T=%g dtype=%d)", N, C, K,
                      (double)inv_T, qk_dtype);
    if (!aligned(workspace, 256)) return refuse(who, MOCO_ERR_INVALID, "workspace must be 256-byte aligned");
    if (!aligned(q, 16) || !aligned(queue_bf16, 16) || !aligned(enq.queue_f32, 16) || !aligned(enq.k_all, 16))
        return refuse(who, MOCO_ERR_INVALID, "q, the queue and k_all must be 16-byte aligned (q=%p queue=%p "
                      "queue_f32=%p k_all=%p)", q, queue_bf16, static_cast<const void*>(enq.queue_f32), enq.k_all);
    NceWorkspace ws = carve_workspace(workspace, N, C);
    if (workspace_bytes < ws.bytes)
        return refuse(who, MOCO_ERR_WORKSPACE, "workspace too small (%zu < %zu)", workspace_bytes, ws.bytes);
    DevInfo d = device_info();
    if (!d.ok) return refuse(who, MOCO_ERR_CUDA, "no CUDA device");
    const __nv_bfloat16* queue = static_cast<const __nv_bfloat16*>(queue_bf16);
    const bool tc = tc_available(d, C);
    const bool want_tc = !(flags & MOCO_NCE_FORCE_SIMT);
    if ((flags & (MOCO_NCE_CTA_PAIR | MOCO_NCE_SINGLE_CTA)) && !tc)
        return refuse(who, MOCO_ERR_UNSUPPORTED, "tensor-core path requested but unavailable (C=%d, sm_%d%d)", C, d.major,
                      d.minor);
    cudaError_t e;
    bool prepped = false;
    // ---- one sweep over the queue for loss + gradient, then ONE tail kernel (merge, dq, optional enqueue)
    const bool one_pass = want_tc && tc && dq && !logits && !(flags & MOCO_NCE_TWO_PASS) &&
                          ((flags & MOCO_NCE_ONE_PASS) || inv_T <= MOCO_ONE_PASS_MAX_INV_T) &&
                          !(normalize && C > 128);
    if (one_pass) {
        const __nv_bfloat16* qb = static_cast<const __nv_bfloat16*>(q);
        if (C > 128 && qk_dtype == MOCO_F32) {            // the C > 128 kernel reads a bf16 copy of q
            e = launch_prep(q, k, qk_dtype, N, C, ws, stream);
            if (e != cudaSuccess) return cuda_result(e, "prep kernel");
            prepped = true;
            qb = ws.q_bf16;
        }
        int slices = 0, n_pad = 0;
        prof_mark(MOCO_PROF_DQ, 0, stream);
        e = launch_sweep(q, qk_dtype, normalize, qb, queue, N, C, K, inv_T, nullptr, d.sms, &slices, &n_pad, ws, stream);
        prof_mark(MOCO_PROF_DQ, 1, stream);
        if (e == cudaSuccess) {
            const bool fuse_enq = enq.n_all > 0 && nce_tail_can_enqueue(C, normalize);
            e = launch_nce_tail(N, C, K, slices, n_pad, inv_T, q, k, qk_dtype, normalize, queue, lse, loss_rows, prob_rows,
                                loss_prob, dq, ws, static_cast<__nv_bfloat16*>(enq.queue_bf16), enq.queue_f32, enq.k_all,
                                enq.k_dtype, fuse_enq ? enq.n_all : 0, enq.index, enq.index_dev, 0, K, stream);
            if (e != cudaSuccess) return cuda_result(e, "tail kernel");
            return fuse_enq ? MOCO_OK : nce_enqueue(enq, C, K, ws, stream);
        }
        if (e != cudaErrorNotSupported) return cuda_result(e, "one-sweep kernel");
        // shape outside the one-sweep kernels' envelope: two-pass below
    }
    if (normalize)
        return refuse(who, MOCO_ERR_UNSUPPORTED, "in-kernel normalisation needs the one-sweep path (C in {64, 128}, N <= "
                      "128 * #SM, gradient requested, no dense logits, inv_T <= %g)", (double)MOCO_ONE_PASS_MAX_INV_T);
    if (!prepped) {
        e = launch_prep(q, k, qk_dtype, N, C, ws, stream);
        if (e != cudaSuccess) return cuda_result(e, "prep kernel");
    }
    const __nv_bfloat16* qb = qk_dtype == MOCO_BF16 ? static_cast<const __nv_bfloat16*>(q) : ws.q_bf16;
    if (want_tc && tc) {
        NceTcParams p = tc_params(qb, queue, N, C, K, inv_T, logits, flags, d.sms);
        prof_mark(MOCO_PROF_STATS, 0, stream);
        e = launch_nce_tc(p, ws, stream);
        prof_mark(MOCO_PROF_STATS, 1, stream);
        if (e == cudaSuccess) {
            e = launch_combine(N, C, p.slices, p.n_pad, inv_T, logits, K, lse, loss_rows, prob_rows, loss_prob, ws, stream);
            if (e != cudaSuccess) return cuda_result(e, "combine kernel");
            if (dq) {
                int slices = 0, n_pad = 0;
                prof_mark(MOCO_PROF_DQ, 0, stream);
                e = launch_sweep(qb, MOCO_BF16, 0, qb, queue, N, C, K, inv_T, lse, d.sms, &slices, &n_pad, ws, stream);
                prof_mark(MOCO_PROF_DQ, 1, stream);
                if (e != cudaSuccess) return cuda_result(e, "dq kernel");
                e = launch_dq_reduce(N, C, slices, n_pad, inv_T, k, qk_dtype, prob_rows, dq, ws.part_o, stream);
                if (e != cudaSuccess) return cuda_result(e, "dq reduce kernel");
            }
            return nce_enqueue(enq, C, K, ws, stream);
        }
        if (e != cudaErrorNotSupported || (flags & (MOCO_NCE_CTA_PAIR | MOCO_NCE_SINGLE_CTA)))
            return cuda_result(e, "statistics kernel");
        // shape outside the tensor-core kernel's envelope (e.g. N > 128 * #SM): generic path below
    }
    e = launch_simt_rows(qb, k, qk_dtype, queue, N, C, K, inv_T, logits, lse, loss_rows, prob_rows, loss_prob, dq, ws, stream);
    if (e != cudaSuccess) return cuda_result(e, "generic NCE kernel");
    return nce_enqueue(enq, C, K, ws, stream);
}

// moco_queue_enqueue (the whole ring, rows [0, K)) and moco_queue_enqueue_shard (the ring rows [row0, row0 + rows)
// this rank holds); `dst` names the destination in the messages
static int queue_enqueue(const char* fn, const char* dst, void* dst_bf16, float* dst_f32, const void* k_all, int k_dtype,
                         int n_all, int C, int64_t K, int64_t index, int64_t row0, int64_t rows, void* stream_) {
    g_err[0] = 0;
    if (!dst_bf16 || !k_all || n_all < 0 || C <= 0 || K <= 0 || index < 0 || index >= K || row0 < 0 || rows <= 0 ||
        row0 + rows > K)
        return refuse(fn, MOCO_ERR_INVALID, "bad argument (n_all=%d C=%d K=%lld index=%lld)", n_all, C, (long long)K,
                      (long long)index);
    if (n_all > K)
        return refuse(fn, MOCO_ERR_INVALID, "n_all (%d) > K (%lld): write order would be ambiguous", n_all,
                      (long long)K);
    if (!aligned(dst_bf16, 16) || !aligned(dst_f32, 16) || !aligned(k_all, 16))
        return refuse(fn, MOCO_ERR_INVALID, "the %s and k_all must be 16-byte aligned (%s=%p %s_f32=%p k_all=%p)", dst,
                      dst, dst_bf16, dst, static_cast<void*>(dst_f32), k_all);
    return cuda_result(launch_enqueue(static_cast<__nv_bfloat16*>(dst_bf16), dst_f32, k_all, k_dtype, n_all, C, K, index,
                                      row0, rows, static_cast<cudaStream_t>(stream_)),
                       "enqueue kernel");
}

// the checks moco_nce_shard_stats and moco_nce_shard_dq share, before their own
static int shard_common(const char* fn, const void* q, int N, int C, int Ks, void* workspace, size_t bytes,
                        NceWorkspace* ws, DevInfo* d) {
    if (!q || !workspace || N <= 0 || C <= 0 || Ks <= 0 || !aligned(workspace, 256))
        return refuse(fn, MOCO_ERR_INVALID, "bad argument");
    *ws = carve_workspace(workspace, N, C);
    if (bytes < ws->bytes) return refuse(fn, MOCO_ERR_WORKSPACE, "workspace too small (%zu < %zu)", bytes, ws->bytes);
    *d = device_info();
    if (!tc_available(*d, C))
        return refuse(fn, MOCO_ERR_UNSUPPORTED, "needs an sm_90 device and C %% 64 == 0, C <= 256 (C=%d)", C);
    return MOCO_OK;
}

// moco_maxpool3x3s2_bwd and (sum: dy2 is required) moco_maxpool3x3s2_bwd2
static int maxpool_bwd(const char* fn, bool sum, const void* dy, const void* dy2, const void* taps, void* dx, int N,
                       int H, int W, int C, void* stream_) {
    g_err[0] = 0;
    if (!ptr16(dy) || (sum && !ptr16(dy2)) || !ptr16(dx) || !taps || !aligned(taps, 8))
        return refuse(fn, MOCO_ERR_INVALID, "null or misaligned pointer");
    return cuda_result(launch_maxpool_bwd(dy, dy2, taps, dx, N, H, W, C, static_cast<cudaStream_t>(stream_)),
                       "max-pool backward kernel", "%s: needs N, H, W >= 1 and C %% 8 == 0 (C=%d)", fn, C);
}

// moco_crop_to_nhwc_bf16 and (src_rows: the images to take) moco_crop_gather_nhwc_bf16
static int crop_to_nhwc(const char* fn, const void* src, int src_dtype, long long src_image_stride,
                        const int64_t* src_rows, void* dst, int N, int C, int HW, void* stream_) {
    g_err[0] = 0;
    if (N < 0 || !dst || (!src && N) || (src_dtype != MOCO_F32 && src_dtype != MOCO_BF16) ||
        src_image_stride < (long long)C * HW || !aligned(src, 16) || !aligned(dst, 16) ||
        (src_image_stride & (src_dtype == MOCO_F32 ? 3 : 7)) != 0)
        return refuse(fn, MOCO_ERR_INVALID, "bad argument");
    return cuda_result(launch_crop_to_nhwc(src, src_dtype, src_image_stride, static_cast<__nv_bfloat16*>(dst), N, C, HW,
                                           static_cast<cudaStream_t>(stream_), src_rows),
                       "crop->nhwc kernel", "%s: needs C <= 4 and H*W %% 8 == 0 (C=%d HW=%d)", fn, C, HW);
}

// moco_shuffle_gather and (pads != nullptr: the cross-GPU barrier of `epoch` before the pull) moco_shuffle_gather_sync
static int shuffle_gather(const char* fn, const void* const* peers, int world, int rows_per_rank, const int64_t* src_rows,
                          int n_rows, size_t row_bytes, void* dst, int flags, void* stream_, void* const* pads, int rank,
                          uint32_t epoch) {
    g_err[0] = 0;
    if (!peers || !src_rows || !dst || world < 1 || world > 16 || rows_per_rank < 1 || n_rows < 0 || row_bytes == 0 ||
        (row_bytes & 15) != 0 || !aligned(dst, 16))
        return refuse(fn, MOCO_ERR_INVALID, "bad argument (world=%d rows_per_rank=%d n_rows=%d row_bytes=%zu)", world,
                      rows_per_rank, n_rows, row_bytes);
    for (int i = 0; i < world; ++i)
        if (!ptr16(peers[i])) return refuse(fn, MOCO_ERR_INVALID, "peer %d pointer null or misaligned", i);
    return cuda_result(launch_gather(peers, world, rows_per_rank, src_rows, n_rows, row_bytes, dst, flags,
                                     static_cast<cudaStream_t>(stream_), pads, rank, epoch),
                       "shuffle gather kernel");
}

extern "C" {

int moco_nce_fwd(const void* q, const void* k, int qk_dtype, const void* queue_bf16, int N, int C, int K,
                 float inv_T, float* logits, float* lse, float* loss_rows, float* prob_rows, float* loss_prob,
                 float* dq, void* workspace, size_t workspace_bytes, int flags, void* stream_) {
    const EnqueueSpec none = {nullptr, nullptr, nullptr, 0, 0, 0, nullptr};
    return nce_head(q, k, qk_dtype, 0, queue_bf16, N, C, K, inv_T, logits, lse, loss_rows, prob_rows, loss_prob, dq,
                    workspace, workspace_bytes, flags, none, static_cast<cudaStream_t>(stream_), "moco_nce_fwd");
}

int moco_nce_step(const void* q, const void* k, int qk_dtype, int normalize, void* queue_bf16, float* queue_f32,
                  int N, int C, int K, float inv_T, const void* k_all, int k_all_dtype, int n_all, int64_t index,
                  int64_t* index_dev, float* lse, float* loss_rows, float* prob_rows, float* loss_prob, float* dq,
                  void* workspace, size_t workspace_bytes, int flags, void* stream_) {
    if (!k_all || n_all < 0 || n_all > K || (k_all_dtype != MOCO_F32 && k_all_dtype != MOCO_BF16) ||
        (!index_dev && (index < 0 || index >= K)))
        return refuse("moco_nce_step", MOCO_ERR_INVALID, "bad enqueue argument (n_all=%d K=%d index=%lld)", n_all, K,
                      (long long)index);
    const EnqueueSpec enq = {queue_bf16, queue_f32, k_all, k_all_dtype, n_all, (long long)index,
                             reinterpret_cast<long long*>(index_dev)};
    return nce_head(q, k, qk_dtype, normalize ? 1 : 0, queue_bf16, N, C, K, inv_T, nullptr, lse, loss_rows, prob_rows,
                    loss_prob, dq, workspace, workspace_bytes, flags, enq, static_cast<cudaStream_t>(stream_),
                    "moco_nce_step");
}

int moco_prof_sweep_window(const void* workspace, int n_ctas, float* us_out, void* stream_) {
    g_err[0] = 0;
    if (!workspace || !us_out || n_ctas < 1 || n_ctas > kMaxCtas)
        return refuse("moco_prof_sweep_window", MOCO_ERR_INVALID, "bad argument");
    NceWorkspace ws = carve_workspace(const_cast<void*>(workspace), 1, 64);
    static unsigned long long host[kMaxCtas * 2];
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    cudaError_t e = cudaMemcpyAsync(host, ws.cta_times, (size_t)n_ctas * 16, cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) return cuda_result(e, "moco_prof_sweep_window");
    unsigned long long lo = ~0ull, hi = 0ull;
    for (int i = 0; i < n_ctas; ++i) {
        if (host[2 * i] == 0ull) continue;
        if (host[2 * i] < lo) lo = host[2 * i];
        if (host[2 * i + 1] > hi) hi = host[2 * i + 1];
    }
    *us_out = (hi > lo) ? (float)((double)(hi - lo) * 1e-3) : 0.f;
    return MOCO_OK;
}

int moco_prof_set_events(int kernel, void* ev_start, void* ev_stop) {
    g_err[0] = 0;
    if (kernel < 0 || kernel > 2) return refuse("moco_prof_set_events", MOCO_ERR_INVALID, "bad kernel id");
    g_prof_ev[kernel][0] = static_cast<cudaEvent_t>(ev_start);
    g_prof_ev[kernel][1] = static_cast<cudaEvent_t>(ev_stop);
    return MOCO_OK;
}

int moco_nce_bwd_dense(const float* grad_logits, const void* k, int k_dtype, const void* queue_bf16, int N, int C,
                       int K, float inv_T, float* dq, void* stream_) {
    g_err[0] = 0;
    if (!grad_logits || !k || !queue_bf16 || !dq || N <= 0 || C <= 0 || K <= 0)
        return refuse("moco_nce_bwd_dense", MOCO_ERR_INVALID, "bad argument");
    return cuda_result(launch_bwd_dense(grad_logits, k, k_dtype, static_cast<const __nv_bfloat16*>(queue_bf16), N, C, K,
                                        inv_T, dq, static_cast<cudaStream_t>(stream_)),
                       "dense backward kernel");
}

int moco_queue_enqueue(void* queue_bf16, float* queue_f32, const void* k_all, int k_dtype, int n_all, int C,
                       int64_t K, int64_t index, void* stream_) {
    return queue_enqueue("moco_queue_enqueue", "queue", queue_bf16, queue_f32, k_all, k_dtype, n_all, C, K, index, 0, K,
                         stream_);
}

// ---------------------------------------------------------------------------------------------------------
// Sharded queue (BASELINE configs[3]): every rank holds rows [shard_row0, shard_row0 + shard_rows) of the ring
// ---------------------------------------------------------------------------------------------------------
int moco_queue_enqueue_shard(void* shard_bf16, float* shard_f32, const void* k_all, int k_dtype, int n_all, int C,
                             int64_t K, int64_t index, int64_t shard_row0, int64_t shard_rows, void* stream_) {
    return queue_enqueue("moco_queue_enqueue_shard", "shard", shard_bf16, shard_f32, k_all, k_dtype, n_all, C, K, index,
                         shard_row0, shard_rows, stream_);
}

int moco_nce_shard_stats(const void* q_all, const void* k_all, int qk_dtype, const void* shard_bf16, int N, int C,
                         int Ks, float inv_T, void* ms_out, void* workspace, size_t workspace_bytes, int flags,
                         void* stream_) {
    g_err[0] = 0;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    NceWorkspace ws; DevInfo d;
    int rc = shard_common("moco_nce_shard_stats", q_all, N, C, Ks, workspace, workspace_bytes, &ws, &d);
    if (rc != MOCO_OK) return rc;
    if (!k_all || !shard_bf16 || !ms_out) return refuse("moco_nce_shard_stats", MOCO_ERR_INVALID, "null pointer");
    cudaError_t e = launch_prep(q_all, k_all, qk_dtype, N, C, ws, stream);
    if (e != cudaSuccess) return cuda_result(e, "prep kernel");
    const __nv_bfloat16* qb = qk_dtype == MOCO_BF16 ? static_cast<const __nv_bfloat16*>(q_all) : ws.q_bf16;
    NceTcParams p = tc_params(qb, shard_bf16, N, C, Ks, inv_T, nullptr, flags, d.sms);
    ShardExact exact = {nullptr, p.q_bf16, p.queue, Ks, inv_T};
    if (flags & MOCO_NCE_ONE_PASS) {
        // one sweep over the shard: (stabiliser, sum) partials for the cross-rank merge AND the unnormalised
        // P~.Queue partials, which stay in the workspace until moco_nce_shard_dq(..., MOCO_NCE_ONE_PASS) rescales them;
        // rows outside the sweep's safe range are evaluated exactly by the combine kernel (and by the dq call)
        e = launch_sweep(q_all, qk_dtype, 0, p.q_bf16, p.queue, N, C, Ks, inv_T, nullptr, d.sms, &p.slices, &p.n_pad, ws, stream);
        if (e != cudaSuccess) return cuda_result(e, "one-pass kernel");
        exact.row_exact = ws.row_exact;
    } else {
        e = launch_nce_tc(p, ws, stream);
        if (e != cudaSuccess) return cuda_result(e, "statistics kernel");
    }
    return cuda_result(launch_combine_partial(N, C, p.slices, p.n_pad, static_cast<float2*>(ms_out), ws, exact, stream),
                       "combine kernel");
}

int moco_nce_shard_merge(const void* ms_all, int world, int N, int C, float inv_T, float* lse, float* loss_rows,
                         float* prob_rows, float* loss_prob, void* workspace, size_t workspace_bytes, void* stream_) {
    g_err[0] = 0;
    if (!ms_all || !lse || !loss_rows || !prob_rows || !loss_prob || !workspace || world < 1 || world > kMaxCtas || N <= 0)
        return refuse("moco_nce_shard_merge", MOCO_ERR_INVALID, "bad argument (null pointer, N=%d, or world=%d outside "
                      "[1, %d])", N, world, kMaxCtas);
    NceWorkspace ws = carve_workspace(workspace, N, C);
    if (workspace_bytes < ws.bytes) return refuse("moco_nce_shard_merge", MOCO_ERR_WORKSPACE, "workspace too small");
    return cuda_result(launch_combine_merge(N, world, inv_T, static_cast<const float2*>(ms_all), lse, loss_rows,
                                            prob_rows, loss_prob, ws, static_cast<cudaStream_t>(stream_)),
                       "combine kernel");
}

int moco_nce_shard_dq(const void* q_all, int q_dtype, const void* shard_bf16, const float* lse_all, int N, int C,
                      int Ks, float inv_T, float* o_partial, void* workspace, size_t workspace_bytes, int flags,
                      void* stream_) {
    g_err[0] = 0;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    NceWorkspace ws; DevInfo d;
    int rc = shard_common("moco_nce_shard_dq", q_all, N, C, Ks, workspace, workspace_bytes, &ws, &d);
    if (rc != MOCO_OK) return rc;
    if (!shard_bf16 || !lse_all || !o_partial) return refuse("moco_nce_shard_dq", MOCO_ERR_INVALID, "null pointer");
    // q_bf16 in the workspace was produced by moco_nce_shard_stats on the same workspace (fp32 inputs)
    const __nv_bfloat16* qb = q_dtype == MOCO_BF16 ? static_cast<const __nv_bfloat16*>(q_all) : ws.q_bf16;
    int slices = 0, n_pad = 0;
    cudaError_t e;
    if (flags & MOCO_NCE_ONE_PASS) {
        // the sweep already happened in moco_nce_shard_stats(..., MOCO_NCE_ONE_PASS) on this workspace: only the
        // slice count is needed, then O = sum_s 2^(m_s - lse) O~_s (exactly, for the rows that call flagged)
        e = launch_sweep(q_all, q_dtype, 0, qb, static_cast<const __nv_bfloat16*>(shard_bf16), N, C, Ks, inv_T, nullptr, d.sms,
                         &slices, &n_pad, ws, stream, /*plan_only=*/true);
        if (e != cudaSuccess) return cuda_result(e, "one-pass plan");
        const ShardExact exact = {ws.row_exact, qb, static_cast<const __nv_bfloat16*>(shard_bf16), Ks, inv_T};
        return cuda_result(launch_dq_reduce(N, C, slices, n_pad, inv_T, nullptr, 0, nullptr, o_partial, ws.part_o, stream,
                                            ws.part_ms, lse_all, exact),
                           "dq reduce kernel");
    }
    e = launch_sweep(q_all, q_dtype, 0, qb, static_cast<const __nv_bfloat16*>(shard_bf16), N, C, Ks, inv_T, lse_all, d.sms, &slices,
                     &n_pad, ws, stream);
    if (e != cudaSuccess) return cuda_result(e, "dq kernel");
    return cuda_result(launch_dq_reduce(N, C, slices, n_pad, inv_T, nullptr, 0, nullptr, o_partial, ws.part_o, stream),
                       "dq reduce kernel");
}

int moco_nce_shard_dq_finish(const float* o_own, const void* k_own, int k_dtype, const float* prob_rows_own, int N,
                             int C, float inv_T, float* dq, void* stream_) {
    g_err[0] = 0;
    if (!o_own || !k_own || !prob_rows_own || !dq || N <= 0 || C <= 0)
        return refuse("moco_nce_shard_dq_finish", MOCO_ERR_INVALID, "bad argument");
    return cuda_result(launch_dq_reduce(N, C, 1, N, inv_T, k_own, k_dtype, prob_rows_own, dq, o_own,
                                        static_cast<cudaStream_t>(stream_)),
                       "dq finish kernel");
}

int moco_nce_shard_dq_finish_peers(const void* const* o_peers_host, int world, int rank, const void* k_own, int k_dtype,
                                   const float* prob_rows_own, int N, int C, float inv_T, float* dq, void* stream_) {
    g_err[0] = 0;
    if (!o_peers_host || !k_own || !prob_rows_own || !dq || N <= 0 || C <= 0 || (C & 3) || world < 1 || world > 16 ||
        rank < 0 || rank >= world)
        return refuse("moco_nce_shard_dq_finish_peers", MOCO_ERR_INVALID, "bad argument (null pointer, N=%d, C=%d not a "
                      "multiple of 4, or world=%d / rank=%d outside 1 <= world <= 16, 0 <= rank < world)", N, C, world,
                      rank);
    for (int r = 0; r < world; ++r)
        if (!ptr16(o_peers_host[r]))
            return refuse("moco_nce_shard_dq_finish_peers", MOCO_ERR_INVALID, "peer %d pointer null or misaligned", r);
    return cuda_result(launch_dq_finish_peers(o_peers_host, world, rank, N, C, inv_T, k_own, k_dtype, prob_rows_own, dq,
                                              static_cast<cudaStream_t>(stream_)),
                       "dq finish (peers) kernel");
}

int moco_f32_to_bf16(const float* src, void* dst, size_t n, void* stream_) {
    g_err[0] = 0;
    if ((!src || !dst) && n) return refuse("moco_f32_to_bf16", MOCO_ERR_INVALID, "null pointer");
    return cuda_result(launch_f32_to_bf16(src, static_cast<__nv_bfloat16*>(dst), n, static_cast<cudaStream_t>(stream_)),
                       "f32->bf16 kernel");
}

int moco_ema_chunk_elems(void) { return ema_chunk_elems(); }

int moco_ema_update(const void* segs, const int32_t* chunk_prefix, int n_segs, int n_chunks, float m, float one_minus_m,
                    void* stream_) {
    g_err[0] = 0;
    if (n_segs < 0 || n_chunks < 0 || ((!segs || !chunk_prefix) && n_segs > 0))
        return refuse("moco_ema_update", MOCO_ERR_INVALID, "bad argument");
    return cuda_result(launch_ema(segs, chunk_prefix, n_segs, n_chunks, m, one_minus_m, static_cast<cudaStream_t>(stream_)),
                       "ema kernel");
}

int moco_crop_s2d_bf16(const void* src, int src_dtype, long long src_image_stride, const int64_t* src_rows, void* dst, int N,
                       int H, int W, void* stream_) {
    g_err[0] = 0;
    if (N < 0 || !dst || (!src && N) || (src_dtype != MOCO_F32 && src_dtype != MOCO_BF16) || src_image_stride < 3LL * H * W ||
        !aligned(src, 8) || !aligned(dst, 16) || (src_image_stride & 1) != 0)
        return refuse("moco_crop_s2d_bf16", MOCO_ERR_INVALID, "bad argument");
    return cuda_result(launch_crop_to_s2d(src, src_dtype, src_image_stride, static_cast<__nv_bfloat16*>(dst), N, H, W,
                                          static_cast<cudaStream_t>(stream_), src_rows),
                       "crop->space-to-depth kernel", "moco_crop_s2d_bf16: needs even H, W >= 2 (H=%d W=%d)", H, W);
}

int moco_augment_crops(const void* pixels, size_t pixels_bytes, const moco_aug_crop* crops, int n_crops, int out_h,
                       int out_w, const float* norm, void* dst, int dst_dtype, float* crop_means, void* stream_) {
    g_err[0] = 0;
    static_assert(sizeof(moco_aug_crop) == 56, "moco_aug_crop is 14 32-bit words ([2N, 14] int32 on the host side)");
    if (!norm || (dst_dtype != MOCO_F32 && dst_dtype != MOCO_BF16) ||
        (n_crops > 0 && (!pixels || pixels_bytes == 0 || !crops || !dst || !crop_means || !aligned(crops, 8) ||
                         !aligned(crop_means, 4) || !aligned(dst, dst_dtype == MOCO_F32 ? 4 : 2))))
        return refuse("moco_augment_crops", MOCO_ERR_INVALID, "bad argument (null or misaligned pointer, empty pixel "
                      "buffer, or dst_dtype=%d)", dst_dtype);
    for (int k = 0; k < 6; ++k)
        if (!isfinite(norm[k]) || (k >= 3 && norm[k] == 0.f))
            return refuse("moco_augment_crops", MOCO_ERR_INVALID, "norm must be finite mean[3], std[3] with std != 0");
    if (!augment_shape_ok(n_crops, out_h, out_w))
        return refuse("moco_augment_crops", MOCO_ERR_INVALID, "needs n_crops in [0, 65535] and out_h, out_w in [1, 1024] "
                      "(n_crops=%d out_h=%d out_w=%d)", n_crops, out_h, out_w);
    return cuda_result(launch_augment(pixels, pixels_bytes, crops, n_crops, out_h, out_w, norm, dst, dst_dtype, crop_means,
                                      static_cast<cudaStream_t>(stream_)),
                       "augment kernels");
}

int moco_augment_crops_blur(const void* pixels, size_t pixels_bytes, const moco_aug_crop_blur* crops, int n_crops,
                            int out_h, int out_w, int ksize, const float* norm, void* dst, int dst_dtype,
                            float* crop_means, void* stream_) {
    g_err[0] = 0;
    static_assert(sizeof(moco_aug_crop_blur) == 128, "moco_aug_crop_blur is 32 32-bit words ([n, 32] int32 on the host)");
    const char* fn = "moco_augment_crops_blur";
    if (!norm || (dst_dtype != MOCO_F32 && dst_dtype != MOCO_BF16) ||
        (n_crops > 0 && (!pixels || pixels_bytes == 0 || !crops || !dst || !crop_means || !aligned(crops, 8) ||
                         !aligned(crop_means, 4) || !aligned(dst, dst_dtype == MOCO_F32 ? 4 : 2))))
        return refuse(fn, MOCO_ERR_INVALID, "bad argument (null or misaligned pointer, empty pixel buffer, or "
                      "dst_dtype=%d)", dst_dtype);
    for (int k = 0; k < 6; ++k)
        if (!isfinite(norm[k]) || (k >= 3 && norm[k] == 0.f))
            return refuse(fn, MOCO_ERR_INVALID, "norm must be finite mean[3], std[3] with std != 0");
    if (!augment_blur_shape_ok(n_crops, out_h, out_w, ksize))
        return refuse(fn, MOCO_ERR_INVALID, "needs n_crops in [0, 65535], out_h, out_w in [1, 512] and an odd ksize in "
                      "[3, 31] with ksize / 2 < min(out_h, out_w) (n_crops=%d out_h=%d out_w=%d ksize=%d)", n_crops,
                      out_h, out_w, ksize);
    return cuda_result(launch_augment_blur(pixels, pixels_bytes, crops, n_crops, out_h, out_w, ksize, norm, dst,
                                           dst_dtype, crop_means, static_cast<cudaStream_t>(stream_)),
                       "augment kernels");
}

int moco_resize_center_crops(const void* pixels, size_t pixels_bytes, const moco_resize_window* windows, int n,
                             int out_h, int out_w, const float* norm, void* dst, int dst_dtype, void* stream_) {
    g_err[0] = 0;
    static_assert(sizeof(moco_resize_window) == 32, "moco_resize_window is 8 32-bit words ([n, 8] int32 on the host)");
    const char* fn = "moco_resize_center_crops";
    if (!norm || (dst_dtype != MOCO_F32 && dst_dtype != MOCO_BF16) ||
        (n > 0 && (!pixels || pixels_bytes == 0 || !windows || !dst || !aligned(windows, 8) ||
                   !aligned(dst, dst_dtype == MOCO_F32 ? 4 : 2))))
        return refuse(fn, MOCO_ERR_INVALID, "bad argument (null or misaligned pointer, empty pixel buffer, or "
                      "dst_dtype=%d)", dst_dtype);
    for (int k = 0; k < 6; ++k)
        if (!isfinite(norm[k]) || (k >= 3 && norm[k] == 0.f))
            return refuse(fn, MOCO_ERR_INVALID, "norm must be finite mean[3], std[3] with std != 0");
    if (!augment_shape_ok(n, out_h, out_w))
        return refuse(fn, MOCO_ERR_INVALID, "needs n in [0, 65535] and out_h, out_w in [1, 1024] (n=%d out_h=%d "
                      "out_w=%d)", n, out_h, out_w);
    return cuda_result(launch_resize_windows(pixels, pixels_bytes, windows, n, out_h, out_w, norm, dst, dst_dtype,
                                             static_cast<cudaStream_t>(stream_)),
                       "resize window kernel");
}

int moco_maxpool3x3s2_fwd(const void* x, void* y, void* taps, int N, int H, int W, int C, void* stream_) {
    g_err[0] = 0;
    if (!ptr16(x) || !ptr16(y) || !taps || !aligned(taps, 8))
        return refuse("moco_maxpool3x3s2_fwd", MOCO_ERR_INVALID, "null or misaligned pointer");
    return cuda_result(launch_maxpool_fwd(x, y, taps, N, H, W, C, static_cast<cudaStream_t>(stream_)),
                       "max-pool forward kernel", "moco_maxpool3x3s2_fwd: needs N, H, W >= 1 and C %% 8 == 0 (C=%d)", C);
}

int moco_maxpool3x3s2_bwd(const void* dy, const void* taps, void* dx, int N, int H, int W, int C, void* stream_) {
    return maxpool_bwd("moco_maxpool3x3s2_bwd", false, dy, nullptr, taps, dx, N, H, W, C, stream_);
}

int moco_maxpool3x3s2_bwd2(const void* dy, const void* dy2, const void* taps, void* dx, int N, int H, int W, int C,
                           void* stream_) {
    return maxpool_bwd("moco_maxpool3x3s2_bwd2", true, dy, dy2, taps, dx, N, H, W, C, stream_);
}

size_t moco_bn_workspace_bytes(void) { return bn_workspace_bytes(); }

static bool bn_layer_fwd_ok(const moco_bn_layer* b) {
    return b && b->gamma && b->beta && b->save_mean && b->save_invstd &&
           (b->running_mean == nullptr) == (b->running_var == nullptr) && b->eps > 0.f;
}

static bool bn_layer_bwd_ok(const moco_bn_layer* b) {
    return b && b->gamma && b->save_mean && b->save_invstd && b->dgamma && b->dbeta;
}

int moco_bn_fwd_train(const void* x, const void* residual, void* y, long long M, int C, const float* gamma,
                      const float* beta, float* running_mean, float* running_var, long long* num_batches_tracked,
                      float momentum, float eps, int relu, float* save_mean, float* save_invstd, void* workspace,
                      size_t workspace_bytes, void* stream_) {
    g_err[0] = 0;
    const moco_bn_layer bn = {gamma, beta, running_mean, running_var, num_batches_tracked, momentum, eps, save_mean,
                              save_invstd, nullptr, nullptr};
    if (!ptr16(x) || !ptr16(y) || !ptr16(workspace) || !bn_layer_fwd_ok(&bn) || !aligned(residual, 16) || x == y)
        return refuse("moco_bn_fwd_train", MOCO_ERR_INVALID, "bad argument (null / misaligned pointer, in-place, "
                      "eps <= 0)");
    BnFwdPlan f{};
    f.x = x; f.res = residual; f.y = y; f.ws = workspace; f.bn = &bn; f.M = M; f.C = C; f.relu = relu;
    return bn_launch("moco_bn_fwd_train", launch_bn_fwd, f, true, workspace_bytes, stream_);
}

int moco_bn_bwd(const void* dy, const void* x, const void* y, long long M, int C, const float* gamma, const float* beta,
                const float* save_mean, const float* save_invstd, int relu, int has_residual, void* dx, void* dresidual,
                float* dgamma, float* dbeta, void* workspace, size_t workspace_bytes, void* stream_) {
    g_err[0] = 0;
    // the backward only reads the saved statistics
    const moco_bn_layer bn = {gamma, beta, nullptr, nullptr, nullptr, 0.f, 0.f, const_cast<float*>(save_mean),
                              const_cast<float*>(save_invstd), dgamma, dbeta};
    if (!ptr16(dy) || !ptr16(x) || !ptr16(dx) || !ptr16(workspace) || !bn_layer_bwd_ok(&bn) || !beta ||
        (relu && has_residual && !y) || !aligned(y, 16) || !aligned(dresidual, 16))
        return refuse("moco_bn_bwd", MOCO_ERR_INVALID, "bad argument (null / misaligned pointer; y is required with "
                      "relu + residual)");
    BnBwdPlan b{};
    b.dy = dy; b.x = x; b.y = y; b.dx = dx; b.dres = dresidual; b.ws = workspace; b.bn = &bn;
    b.M = M; b.C = C; b.relu = relu; b.has_residual = has_residual;
    return bn_launch("moco_bn_bwd", launch_bn_bwd, b, true, workspace_bytes, stream_);
}

int moco_bn_add_relu_fwd_train(const void* x, const void* residual, void* y, void* mask, long long M, int C,
                               const moco_bn_layer* bn, const moco_bn_layer* shortcut, void* workspace,
                               size_t workspace_bytes, void* stream_) {
    g_err[0] = 0;
    if (!ptr16(x) || !ptr16(residual) || !ptr16(y) || !ptr16(workspace) || !bn_layer_fwd_ok(bn) ||
        (shortcut && !bn_layer_fwd_ok(shortcut)) || x == y || residual == y)
        return refuse("moco_bn_add_relu_fwd_train", MOCO_ERR_INVALID, "bad argument (null / misaligned pointer, "
                      "in-place, eps <= 0, one of running_mean / running_var)");
    BnFwdPlan f{};
    f.x = x; f.res = residual; f.y = y; f.mask = mask; f.ws = workspace; f.bn = bn; f.sc = shortcut;
    f.M = M; f.C = C; f.relu = 1;
    return bn_launch("moco_bn_add_relu_fwd_train", launch_bn_fwd, f, true, workspace_bytes, stream_);
}

int moco_bn_fwd_train_given(const void* x, const void* residual, void* y, void* mask, long long M, int C, int relu,
                            const moco_bn_layer* bn, const moco_bn_layer* shortcut, int stats_given, void* workspace,
                            size_t workspace_bytes, void* stream_) {
    g_err[0] = 0;
    const bool passes = !(stats_given & MOCO_BN_STATS_GIVEN) || (shortcut && !(stats_given & MOCO_BN_SC_STATS_GIVEN));
    if (!ptr16(x) || !ptr16(y) || !bn_layer_fwd_ok(bn) || (shortcut && (!bn_layer_fwd_ok(shortcut) || !residual)) ||
        (stats_given & ~(MOCO_BN_STATS_GIVEN | MOCO_BN_SC_STATS_GIVEN)) || (passes && !workspace) ||
        !aligned(residual, 16) || !aligned(workspace, 16) || x == y || residual == y)
        return refuse("moco_bn_fwd_train_given", MOCO_ERR_INVALID, "bad argument (null / misaligned pointer, in-place, "
                      "eps <= 0, one of running_mean / running_var, unknown stats_given bits; a shortcut BN needs "
                      "residual, a statistics pass the workspace)");
    BnFwdPlan f{};
    f.x = x; f.res = residual; f.y = y; f.mask = mask; f.ws = workspace; f.bn = bn; f.sc = shortcut;
    f.M = M; f.C = C; f.relu = relu; f.given = stats_given;
    return bn_launch("moco_bn_fwd_train_given", launch_bn_fwd, f, passes, workspace_bytes, stream_);
}

size_t moco_conv1x1_workspace_bytes(void) { return conv1x1_workspace_bytes(); }

int moco_conv1x1_bn_stats(const void* x, const void* w, void* y, long long M, int Cin, int Cout,
                          const moco_bn_layer* bn, void* workspace, size_t workspace_bytes, void* stream_) {
    g_err[0] = 0;
    const char* fn = "moco_conv1x1_bn_stats";
    if (!ptr16(x) || !ptr16(w) || !ptr16(y) || !ptr16(workspace) || !bn || !bn->save_mean || !bn->save_invstd ||
        (bn->running_mean == nullptr) != (bn->running_var == nullptr) || !(bn->eps > 0.f) || x == y || w == y)
        return refuse(fn, MOCO_ERR_INVALID, "bad argument (null / misaligned pointer, in-place, eps <= 0, one of "
                      "running_mean / running_var)");
    if (!conv1x1_stats_shape_ok(M, Cin, Cout))
        return refuse(fn, MOCO_ERR_UNSUPPORTED, "needs 1 <= M < 2^31 - 128, Cin a multiple of 64 in [64, 65536] and "
                      "Cout a multiple of 64 in [64, 4096] (M=%lld Cin=%d Cout=%d)", M, Cin, Cout);
    if (workspace_bytes < conv1x1_workspace_bytes()) return refuse(fn, MOCO_ERR_WORKSPACE, "workspace too small");
    return cuda_result(launch_conv1x1_bn_stats(x, w, y, M, Cin, Cout, *bn, workspace, static_cast<cudaStream_t>(stream_)),
                       fn);
}

int moco_conv1x1_bn_add_relu_fwd(const void* x, const void* w, const void* residual, void* y, void* mask, long long M,
                                 int Cin, int Cout, const moco_bn_layer* bn, const moco_bn_layer* shortcut,
                                 int stats_given, void* workspace, size_t workspace_bytes, void* stream_) {
    g_err[0] = 0;
    const char* fn = "moco_conv1x1_bn_add_relu_fwd";
    const bool passes = !(stats_given & MOCO_BN_STATS_GIVEN) || (shortcut && !(stats_given & MOCO_BN_SC_STATS_GIVEN));
    if (!ptr16(x) || !ptr16(w) || !ptr16(residual) || !ptr16(y) || !bn_layer_fwd_ok(bn) ||
        (shortcut && !bn_layer_fwd_ok(shortcut)) || (stats_given & ~(MOCO_BN_STATS_GIVEN | MOCO_BN_SC_STATS_GIVEN)) ||
        (passes && !workspace) || !aligned(workspace, 16) || y == x || y == w || y == residual ||
        (mask && (mask == x || mask == y || mask == residual)))
        return refuse(fn, MOCO_ERR_INVALID, "bad argument (null / misaligned pointer, in-place, eps <= 0, one of "
                      "running_mean / running_var, unknown stats_given bits; a statistics pass needs the workspace)");
    if (!conv1x1_apply_shape_ok(M, Cin, Cout))
        return refuse(fn, MOCO_ERR_UNSUPPORTED, "needs 1 <= M < 2^31 - 128, Cin a multiple of 64 in [64, 65536] and "
                      "Cout a power of two in [64, 2048] (M=%lld Cin=%d Cout=%d)", M, Cin, Cout);
    const size_t need = conv1x1_workspace_bytes() > bn_workspace_bytes() ? conv1x1_workspace_bytes()
                                                                          : bn_workspace_bytes();
    if (passes && workspace_bytes < need)
        return refuse(fn, MOCO_ERR_WORKSPACE, "workspace too small (%zu < %zu)", workspace_bytes, need);
    return cuda_result(launch_conv1x1_bn_add_relu(x, w, residual, y, mask, M, Cin, Cout, *bn, shortcut, stats_given,
                                                  workspace, static_cast<cudaStream_t>(stream_)),
                       fn);
}

int moco_conv1x1_dgrad_bn_bwd(const void* dh, const void* w, void* g, long long M, int Cin, int Cout, const void* x,
                              const void* mask, const void* dy2, const void* x2, const moco_bn_layer* bn,
                              const moco_bn_layer* shortcut, void* workspace, size_t workspace_bytes, void* stream_) {
    g_err[0] = 0;
    const char* fn = "moco_conv1x1_dgrad_bn_bwd";
    if (!ptr16(dh) || !ptr16(w) || !ptr16(g) || !ptr16(x) || !ptr16(workspace) || !bn || !bn->save_mean ||
        !bn->save_invstd || !bn->dgamma || !bn->dbeta || (x2 == nullptr) != (shortcut == nullptr) ||
        !aligned(mask, 16) || !aligned(dy2, 16) || !aligned(x2, 16) || g == dh || g == w || g == x || g == mask ||
        g == dy2)
        return refuse(fn, MOCO_ERR_INVALID, "bad argument (null / misaligned pointer, g aliasing an input, x2 without "
                      "the shortcut BN or the reverse)");
    if (!mask || !dy2 || x2 || !conv1x1_dgrad_shape_ok(M, Cin, Cout))
        return refuse(fn, MOCO_ERR_UNSUPPORTED, "needs the mask bits and dy2 without a shortcut BN, 1 <= M < 2^31 - "
                      "128, Cin a power of two in [128, 2048] and Cout a multiple of 64 in [64, 4096] (M=%lld Cin=%d "
                      "Cout=%d)", M, Cin, Cout);
    if (workspace_bytes < conv1x1_workspace_bytes()) return refuse(fn, MOCO_ERR_WORKSPACE, "workspace too small");
    return cuda_result(launch_conv1x1_dgrad_bn_bwd(dh, w, g, M, Cin, Cout, x, mask, dy2, *bn, workspace,
                                                   static_cast<cudaStream_t>(stream_)),
                       fn);
}

size_t moco_knn_workspace_bytes(int Nq, long long Nb, long long capacity) {
    if (Nq < 1 || Nq > kKnnMaxNq || Nb < 1 || Nb >= (1LL << 31) || capacity < 1 || capacity > Nb) return 0;
    return knn_carve(nullptr, Nq, Nb, capacity).bytes;
}

int moco_knn(const void* q, const void* bank, const int32_t* labels, int Nq, long long Nb, int C, int k, float inv_T,
             int n_classes, const int32_t* targets, int32_t* top5, float* scores5, int32_t* nbr_idx, float* nbr_sim,
             int32_t* correct, void* workspace, size_t workspace_bytes, long long* need_capacity, void* stream_) {
    g_err[0] = 0;
    const char* fn = "moco_knn";
    if (!ptr16(q) || !ptr16(bank) || !labels || !top5 || !workspace || !aligned(workspace, 256) || !need_capacity ||
        (targets == nullptr) != (correct == nullptr) || !aligned(labels, 4) || !aligned(targets, 4) ||
        !aligned(top5, 4) || !aligned(scores5, 4) || !aligned(nbr_idx, 4) || !aligned(nbr_sim, 4) ||
        !aligned(correct, 4))
        return refuse(fn, MOCO_ERR_INVALID, "bad argument (null / misaligned pointer; targets and correct go together)");
    if (!(inv_T > 0.f) || !isfinite(inv_T) || n_classes < 1 || n_classes > 65536 || k < 1 || Nb < k)
        return refuse(fn, MOCO_ERR_INVALID, "needs inv_T > 0 finite, n_classes in [1, 65536] and 1 <= k <= Nb "
                      "(inv_T=%g n_classes=%d k=%d Nb=%lld)", (double)inv_T, n_classes, k, Nb);
    if (!knn_shape_ok(Nq, Nb, C, k))
        return refuse(fn, MOCO_ERR_UNSUPPORTED, "needs 1 <= Nq <= %d, C a multiple of 64 in [64, 2048], k <= 1024 and "
                      "Nb < 2^31 (Nq=%d C=%d k=%d Nb=%lld)", kKnnMaxNq, Nq, C, k, Nb);
    // every output apart from the inputs, the workspace and one another
    struct Buf { const void* p; size_t n; };
    const Buf in[] = {{q, (size_t)Nq * C * 2}, {bank, (size_t)Nb * C * 2}, {labels, (size_t)Nb * 4},
                      {targets, (size_t)Nq * 4}, {workspace, workspace_bytes}};
    const Buf out[] = {{top5, (size_t)Nq * 20}, {scores5, (size_t)Nq * 20}, {nbr_idx, (size_t)Nq * k * 4},
                       {nbr_sim, (size_t)Nq * k * 4}, {correct, 8}};
    auto overlap = [](const Buf& a, const Buf& b) {
        const char *pa = static_cast<const char*>(a.p), *pb = static_cast<const char*>(b.p);
        return a.p && b.p && pa < pb + b.n && pb < pa + a.n;
    };
    for (int i = 0; i < 5; ++i) {
        for (const Buf& b : in)
            if (overlap(out[i], b)) return refuse(fn, MOCO_ERR_INVALID, "output %d overlaps an input or the workspace", i);
        for (int j = 0; j < i; ++j)
            if (overlap(out[i], out[j])) return refuse(fn, MOCO_ERR_INVALID, "outputs %d and %d overlap", j, i);
    }
    KnnWorkspace ws = knn_carve(workspace, Nq, Nb, 0);
    const size_t need = ws.fixed + (size_t)Nq * k * 8;
    if (workspace_bytes < need)
        return refuse(fn, MOCO_ERR_WORKSPACE, "workspace too small (%zu < %zu, a capacity of k candidates per query)",
                      workspace_bytes, need);
    long long cap = (long long)((workspace_bytes - ws.fixed) / ((size_t)Nq * 8));
    if (cap > Nb) cap = Nb;                                // no query has more candidates than the bank has rows
    ws = knn_carve(workspace, Nq, Nb, cap);
    const DevInfo d = device_info();
    if (!d.ok || d.major != 9) return refuse(fn, MOCO_ERR_UNSUPPORTED, "needs an sm_90 device");
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const KnnPlan p = {labels, targets, Nq, Nb, C, k, n_classes, inv_T, top5, scores5, nbr_idx, nbr_sim, correct};
    const int rc = cuda_result(launch_knn(q, bank, p, ws, stream), fn);
    if (rc != MOCO_OK) return rc;
    unsigned int status[2] = {0u, 0u};
    cudaError_t e = cudaMemcpyAsync(status, ws.status, sizeof(status), cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) return cuda_result(e, fn);
    *need_capacity = status[0];                            // the largest candidate count of any query
    if (status[1]) return refuse(fn, MOCO_ERR_INVALID, "a neighbour's label is outside [0, %d)", n_classes);
    if (status[0] > (unsigned long long)cap)
        return refuse(fn, MOCO_ERR_CAPACITY, "a query has %u candidates, the workspace holds %lld", status[0], cap);
    return MOCO_OK;
}

int moco_bn_bwd_apply_given(const void* g, const void* x, const void* x2, long long M, int C, const moco_bn_layer* bn,
                            const moco_bn_layer* shortcut, void* dx, void* dx2, void* stream_) {
    g_err[0] = 0;
    if (!ptr16(g) || !ptr16(x) || !ptr16(dx) || !bn_layer_bwd_ok(bn) ||
        (shortcut && (!bn_layer_bwd_ok(shortcut) || !x2 || !dx2)) || !aligned(x2, 16) || !aligned(dx2, 16))
        return refuse("moco_bn_bwd_apply_given", MOCO_ERR_INVALID, "bad argument (null / misaligned pointer; x2 and dx2 "
                      "are required with a shortcut BN)");
    BnBwdPlan b{};
    b.dy = g; b.x = x; b.x2 = x2; b.dx = dx; b.dres = dx2; b.bn = bn; b.sc = shortcut; b.M = M; b.C = C; b.reduced = 1;
    return bn_launch("moco_bn_bwd_apply_given", launch_bn_bwd, b, false, 0, stream_);
}

// moco_bn_add_relu_bwd and (sum: dy2 is required) moco_bn_add_relu_bwd2
static int bn_add_relu_bwd(const char* fn, bool sum, const void* dy, const void* dy2, const void* x,
                           const void* residual, const void* mask, long long M, int C, const moco_bn_layer* bn,
                           const moco_bn_layer* shortcut, void* dx, void* dresidual, void* workspace,
                           size_t workspace_bytes, void* stream_) {
    g_err[0] = 0;
    if (!ptr16(dy) || (sum && !dy2) || !ptr16(x) || !mask || !ptr16(dx) || !ptr16(workspace) || !bn_layer_bwd_ok(bn) ||
        (shortcut && (!bn_layer_bwd_ok(shortcut) || !residual || !dresidual)) || !aligned(dy2, 16) ||
        !aligned(residual, 16) || !aligned(dresidual, 16))
        return refuse(fn, MOCO_ERR_INVALID, "bad argument (null / misaligned pointer; residual and dresidual are "
                      "required with a shortcut BN)");
    BnBwdPlan b{};
    b.dy = dy; b.dy2 = dy2; b.x = x; b.mbits = mask; b.x2 = residual; b.dx = dx; b.dres = dresidual; b.ws = workspace;
    b.bn = bn; b.sc = shortcut; b.M = M; b.C = C;
    return bn_launch(fn, launch_bn_bwd, b, true, workspace_bytes, stream_);
}

int moco_bn_add_relu_bwd(const void* dy, const void* x, const void* residual, const void* mask, long long M, int C,
                         const moco_bn_layer* bn, const moco_bn_layer* shortcut, void* dx, void* dresidual,
                         void* workspace, size_t workspace_bytes, void* stream_) {
    return bn_add_relu_bwd("moco_bn_add_relu_bwd", false, dy, nullptr, x, residual, mask, M, C, bn, shortcut, dx,
                           dresidual, workspace, workspace_bytes, stream_);
}

int moco_bn_add_relu_bwd2(const void* dy, const void* dy2, const void* x, const void* residual, const void* mask,
                          long long M, int C, const moco_bn_layer* bn, const moco_bn_layer* shortcut, void* dx,
                          void* dresidual, void* workspace, size_t workspace_bytes, void* stream_) {
    return bn_add_relu_bwd("moco_bn_add_relu_bwd2", true, dy, dy2, x, residual, mask, M, C, bn, shortcut, dx,
                           dresidual, workspace, workspace_bytes, stream_);
}

int moco_bn_relu_maxpool_fwd_train(const void* x, void* y, void* taps, int N, int H, int W, int C,
                                   const moco_bn_layer* bn, void* workspace, size_t workspace_bytes, void* stream_) {
    g_err[0] = 0;
    const char* fn = "moco_bn_relu_maxpool_fwd_train";
    if (!ptr16(x) || !ptr16(y) || !taps || !aligned(taps, 8) || !ptr16(workspace) || !bn_layer_fwd_ok(bn))
        return refuse(fn, MOCO_ERR_INVALID, "bad argument (null / misaligned pointer, eps <= 0, one of running_mean / "
                      "running_var)");
    if (workspace_bytes < bn_workspace_bytes()) return refuse(fn, MOCO_ERR_WORKSPACE, "workspace too small");
    return cuda_result(launch_bn_relu_maxpool_fwd(x, y, taps, N, H, W, C, *bn, workspace, static_cast<cudaStream_t>(stream_)),
                       "batch-norm + max-pool forward kernels", "%s: needs N, H, W >= 1 and C a power of two in "
                       "[64, 2048] (C=%d)", fn, C);
}

// the frozen BatchNorm entry points: scale / shift required, the shortcut's pair both or neither (and only with a
// residual to apply it to)
static bool bn_eval_coefs_ok(const float* scale, const float* shift, const void* residual, const float* sc_scale,
                             const float* sc_shift) {
    return scale && shift && (sc_scale == nullptr) == (sc_shift == nullptr) && (sc_scale == nullptr || residual);
}

int moco_bn_eval_act(const void* x, const void* residual, void* y, long long M, int C, const float* scale,
                     const float* shift, int relu, const float* sc_scale, const float* sc_shift, void* stream_) {
    g_err[0] = 0;
    if (!ptr16(x) || !ptr16(y) || !bn_eval_coefs_ok(scale, shift, residual, sc_scale, sc_shift) ||
        !aligned(residual, 16) || x == y || residual == y)
        return refuse("moco_bn_eval_act", MOCO_ERR_INVALID, "bad argument (null / misaligned pointer, in-place, one of "
                      "sc_scale / sc_shift, a shortcut BN without a residual)");
    return cuda_result(launch_bn_eval_act(x, residual, y, M, C, scale, shift, relu, sc_scale, sc_shift,
                                          static_cast<cudaStream_t>(stream_)),
                       "batch-norm eval kernel", "moco_bn_eval_act: needs M >= 1 and C a power of two in [64, 2048] "
                       "(M=%lld C=%d)", M, C);
}

int moco_bn_relu_maxpool_eval(const void* x, void* y, int N, int H, int W, int C, const float* scale,
                              const float* shift, void* stream_) {
    g_err[0] = 0;
    if (!ptr16(x) || !ptr16(y) || !scale || !shift || x == y)
        return refuse("moco_bn_relu_maxpool_eval", MOCO_ERR_INVALID, "bad argument (null / misaligned pointer, "
                      "in-place)");
    return cuda_result(launch_bn_relu_maxpool_eval(x, y, N, H, W, C, scale, shift, static_cast<cudaStream_t>(stream_)),
                       "batch-norm eval + max-pool kernel", "moco_bn_relu_maxpool_eval: needs N, H, W >= 1 and C a "
                       "power of two in [64, 2048] (C=%d)", C);
}

int moco_bn_eval_act_avgpool(const void* x, const void* residual, float* feat, int N, int HW, int C, const float* scale,
                             const float* shift, int relu, const float* sc_scale, const float* sc_shift, void* stream_) {
    g_err[0] = 0;
    if (!ptr16(x) || !ptr16(feat) || !bn_eval_coefs_ok(scale, shift, residual, sc_scale, sc_shift) ||
        !aligned(residual, 16))
        return refuse("moco_bn_eval_act_avgpool", MOCO_ERR_INVALID, "bad argument (null / misaligned pointer, one of "
                      "sc_scale / sc_shift, a shortcut BN without a residual)");
    return cuda_result(launch_bn_eval_act_avgpool(x, residual, feat, N, HW, C, scale, shift, relu, sc_scale, sc_shift,
                                                  static_cast<cudaStream_t>(stream_)),
                       "batch-norm eval + average-pool kernel", "moco_bn_eval_act_avgpool: needs N, HW >= 1 and C a "
                       "power of two in [64, 2048] (N=%d HW=%d C=%d)", N, HW, C);
}

int moco_crop_to_nhwc_bf16(const void* src, int src_dtype, long long src_image_stride, void* dst, int N, int C, int HW,
                           void* stream_) {
    return crop_to_nhwc("moco_crop_to_nhwc_bf16", src, src_dtype, src_image_stride, nullptr, dst, N, C, HW, stream_);
}

int moco_crop_gather_nhwc_bf16(const void* src, int src_dtype, long long src_image_stride, const int64_t* src_rows,
                               void* dst, int N, int C, int HW, void* stream_) {
    return crop_to_nhwc("moco_crop_gather_nhwc_bf16", src, src_dtype, src_image_stride, src_rows, dst, N, C, HW, stream_);
}

int moco_shuffle_gather(const void* const* peers, int world, int rows_per_rank, const int64_t* src_rows, int n_rows,
                        size_t row_bytes, void* dst, int flags, void* stream_) {
    return shuffle_gather("moco_shuffle_gather", peers, world, rows_per_rank, src_rows, n_rows, row_bytes, dst, flags,
                          stream_, nullptr, 0, 0);
}

int moco_shuffle_gather_sync(const void* const* peers, void* const* pads, int world, int rank, uint32_t epoch,
                             int rows_per_rank, const int64_t* src_rows, int n_rows, size_t row_bytes, void* dst,
                             int flags, void* stream_) {
    if (!pads || rank < 0 || rank >= world || epoch == 0)
        return refuse("moco_shuffle_gather_sync", MOCO_ERR_INVALID, "bad synchronisation argument (rank=%d world=%d "
                      "epoch=%u)", rank, world, epoch);
    return shuffle_gather("moco_shuffle_gather_sync", peers, world, rows_per_rank, src_rows, n_rows, row_bytes, dst,
                          flags, stream_, pads, rank, epoch);
}

int moco_p2p_last_timeout(uint32_t out[4]) {
    g_err[0] = 0;
    unsigned int* w = out ? p2p_status_words() : nullptr;
    if (!w) return refuse("moco_p2p_last_timeout", MOCO_ERR_INVALID, "no status block");
    for (int i = 0; i < 4; ++i) out[i] = w[i];
    return MOCO_OK;
}

int moco_signal_barrier(void* const* pads, int world, int rank, uint32_t epoch, void* stream_) {
    g_err[0] = 0;
    if (!pads || world < 1 || world > 16 || rank < 0 || rank >= world)
        return refuse("moco_signal_barrier", MOCO_ERR_INVALID, "bad argument");
    return cuda_result(launch_signal_barrier(pads, world, rank, epoch, static_cast<cudaStream_t>(stream_)),
                       "signal barrier kernel");
}

int moco_p2p_alloc(size_t bytes, void** dev_ptr_out, unsigned char handle_out[64]) {
    g_err[0] = 0;
    if (!dev_ptr_out || !handle_out || bytes == 0) return refuse("moco_p2p_alloc", MOCO_ERR_INVALID, "bad argument");
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) return cuda_result(e, "cudaMalloc");
    e = cudaMemset(p, 0, bytes);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { cudaFree(p); return cuda_result(e, "cudaMemset"); }
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    cudaIpcMemHandle_t h;
    e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) { cudaFree(p); return cuda_result(e, "cudaIpcGetMemHandle"); }
    memcpy(handle_out, &h, 64);
    *dev_ptr_out = p;
    return MOCO_OK;
}

int moco_p2p_open(const unsigned char handle[64], void** dev_ptr_out) {
    g_err[0] = 0;
    if (!handle || !dev_ptr_out) return refuse("moco_p2p_open", MOCO_ERR_INVALID, "bad argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    void* p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return cuda_result(e, "cudaIpcOpenMemHandle");
    *dev_ptr_out = p;
    return MOCO_OK;
}

int moco_p2p_close(void* dev_ptr) {
    g_err[0] = 0;
    return cuda_result(cudaIpcCloseMemHandle(dev_ptr), "cudaIpcCloseMemHandle");
}

int moco_p2p_free(void* dev_ptr) {
    g_err[0] = 0;
    return cuda_result(cudaFree(dev_ptr), "cudaFree");
}

}  // extern "C"
