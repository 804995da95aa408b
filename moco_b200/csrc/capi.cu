// extern "C" boundary of libmoco_b200.so (see include/moco_b200.h).
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include "../../include/moco_b200.h"
#include "common.cuh"

namespace moco {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

static int cuda_fail(const char* what, cudaError_t e) {
    if (e == cudaErrorNotSupported) {
        set_error("%s: shape/device not supported by this kernel", what);
        return MOCO_ERR_UNSUPPORTED;
    }
    if (g_err[0] == 0 || e != cudaErrorUnknown) set_error("%s: %s", what, cudaGetErrorString(e));
    return MOCO_ERR_CUDA;
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

}  // namespace moco

using namespace moco;

extern "C" {

int moco_abi_version(void) { return MOCO_B200_ABI_VERSION; }

const char* moco_last_error(void) { return g_err; }

int moco_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    DevInfo d = device_info();
    if (!d.ok) { set_error("no CUDA device"); return MOCO_ERR_CUDA; }
    if (sm_count) *sm_count = d.sms;
    if (cc_major) *cc_major = d.major;
    if (cc_minor) *cc_minor = d.minor;
    return MOCO_OK;
}

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

struct EnqueueSpec {            // n_all == 0: no enqueue
    void* queue_bf16; float* queue_f32; const void* k_all; int k_dtype; int n_all;
    long long index; long long* index_dev;
};

static int nce_head(const void* q, const void* k, int qk_dtype, int normalize, const void* queue_bf16, int N, int C,
                    int K, float inv_T, float* logits, float* lse, float* loss_rows, float* prob_rows, float* loss_prob,
                    float* dq, void* workspace, size_t workspace_bytes, int flags, const EnqueueSpec& enq,
                    cudaStream_t stream, const char* who) {
    g_err[0] = 0;
    if (!q || !k || !queue_bf16 || !lse || !loss_rows || !prob_rows || !loss_prob || !workspace) {
        set_error("%s: null pointer argument", who);
        return MOCO_ERR_INVALID;
    }
    if (N <= 0 || C <= 0 || K <= 0 || !(inv_T > 0.f) || (qk_dtype != MOCO_F32 && qk_dtype != MOCO_BF16)) {
        set_error("%s: bad N/C/K/inv_T/dtype (N=%d C=%d K=%d inv_T=%g dtype=%d)", who, N, C, K, (double)inv_T, qk_dtype);
        return MOCO_ERR_INVALID;
    }
    if ((reinterpret_cast<uintptr_t>(workspace) & 255) != 0) {
        set_error("%s: workspace must be 256-byte aligned", who);
        return MOCO_ERR_INVALID;
    }
    NceWorkspace ws = carve_workspace(workspace, N, C);
    if (workspace_bytes < ws.bytes) {
        set_error("%s: workspace too small (%zu < %zu)", who, workspace_bytes, ws.bytes);
        return MOCO_ERR_WORKSPACE;
    }
    DevInfo d = device_info();
    if (!d.ok) { set_error("%s: no CUDA device", who); return MOCO_ERR_CUDA; }
    const __nv_bfloat16* queue = static_cast<const __nv_bfloat16*>(queue_bf16);
    const bool aligned = ((reinterpret_cast<uintptr_t>(q) & 15) == 0) && ((reinterpret_cast<uintptr_t>(queue) & 15) == 0);
    const bool tc_shape = (C % 64 == 0) && C <= 256 && aligned;
    const bool want_tc = !(flags & MOCO_NCE_FORCE_SIMT);
    if ((flags & (MOCO_NCE_CTA_PAIR | MOCO_NCE_SINGLE_CTA)) && (!tc_shape || d.major != 9)) {
        set_error("%s: tensor-core path requested but unavailable (C=%d, sm_%d%d)", who, C, d.major, d.minor);
        return MOCO_ERR_UNSUPPORTED;
    }
    cudaError_t e;
    bool prepped = false;
    // ---- one sweep over the queue for loss + gradient, then ONE tail kernel (merge, dq, optional enqueue)
    const bool one_pass = want_tc && tc_shape && d.major == 9 && dq && !logits && !(flags & MOCO_NCE_TWO_PASS) &&
                          ((flags & MOCO_NCE_ONE_PASS) || inv_T <= MOCO_ONE_PASS_MAX_INV_T) &&
                          !(normalize && C > 128);
    if (one_pass) {
        const __nv_bfloat16* qb = static_cast<const __nv_bfloat16*>(q);
        if (C > 128 && qk_dtype == MOCO_F32) {            // the C > 128 kernel reads a bf16 copy of q
            e = launch_prep(q, k, qk_dtype, N, C, ws, stream);
            if (e != cudaSuccess) return cuda_fail("prep kernel", e);
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
            if (e != cudaSuccess) return cuda_fail("tail kernel", e);
            if (enq.n_all > 0 && !fuse_enq) {
                e = launch_enqueue(static_cast<__nv_bfloat16*>(enq.queue_bf16), enq.queue_f32, enq.k_all, enq.k_dtype,
                                   enq.n_all, C, K, enq.index, 0, K, stream);
                if (e != cudaSuccess) return cuda_fail("enqueue kernel", e);
            }
            return MOCO_OK;
        }
        if (e != cudaErrorNotSupported) return cuda_fail("one-sweep kernel", e);
        // shape outside the one-sweep kernels' envelope: two-pass below
    }
    if (normalize || enq.index_dev) {
        set_error("%s: in-kernel normalisation / device-side ring index need the one-sweep path "
                  "(C in {64, 128}, gradient requested, no dense logits, inv_T <= %g)", who, (double)MOCO_ONE_PASS_MAX_INV_T);
        return MOCO_ERR_UNSUPPORTED;
    }
    if (!prepped) {
        e = launch_prep(q, k, qk_dtype, N, C, ws, stream);
        if (e != cudaSuccess) return cuda_fail("prep kernel", e);
    }
    const __nv_bfloat16* qb = qk_dtype == MOCO_BF16 ? static_cast<const __nv_bfloat16*>(q) : ws.q_bf16;
    auto finish = [&]() -> int {                       // the enqueue of moco_nce_step on the non-fused paths
        if (enq.n_all > 0) {
            cudaError_t ee = launch_enqueue(static_cast<__nv_bfloat16*>(enq.queue_bf16), enq.queue_f32, enq.k_all,
                                            enq.k_dtype, enq.n_all, C, K, enq.index, 0, K, stream);
            if (ee != cudaSuccess) return cuda_fail("enqueue kernel", ee);
        }
        return MOCO_OK;
    };
    if (want_tc && tc_shape && d.major == 9) {
        NceTcParams p;
        p.q_bf16 = qb; p.queue = queue; p.N = N; p.C = C; p.K = K; p.inv_T = inv_T; p.logits = logits;
        p.cta_group = (flags & MOCO_NCE_CTA_PAIR) ? 2 : 1;
        p.num_sms = d.sms;
        p.slices = 0; p.n_pad = 0;
        prof_mark(MOCO_PROF_STATS, 0, stream);
        e = launch_nce_tc(p, ws, stream);
        prof_mark(MOCO_PROF_STATS, 1, stream);
        if (e == cudaSuccess) {
            e = launch_combine(N, C, p.slices, p.n_pad, inv_T, logits, K, lse, loss_rows, prob_rows, loss_prob, ws, stream);
            if (e != cudaSuccess) return cuda_fail("combine kernel", e);
            if (dq) {
                int slices = 0, n_pad = 0;
                prof_mark(MOCO_PROF_DQ, 0, stream);
                e = launch_sweep(qb, MOCO_BF16, 0, qb, queue, N, C, K, inv_T, lse, d.sms, &slices, &n_pad, ws, stream);
                prof_mark(MOCO_PROF_DQ, 1, stream);
                if (e != cudaSuccess) return cuda_fail("dq kernel", e);
                e = launch_dq_reduce(N, C, slices, n_pad, inv_T, k, qk_dtype, prob_rows, dq, ws.part_o, stream);
                if (e != cudaSuccess) return cuda_fail("dq reduce kernel", e);
            }
            return finish();
        }
        if (e != cudaErrorNotSupported || (flags & (MOCO_NCE_CTA_PAIR | MOCO_NCE_SINGLE_CTA)))
            return cuda_fail("statistics kernel", e);
        // shape outside the tensor-core kernel's envelope (e.g. N > 128 * #SM): generic path below
    }
    e = launch_simt_rows(qb, k, qk_dtype, queue, N, C, K, inv_T, logits, lse, loss_rows, prob_rows, loss_prob, dq, ws, stream);
    if (e != cudaSuccess) return cuda_fail("generic NCE kernel", e);
    return finish();
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
        (!index_dev && (index < 0 || index >= K))) {
        g_err[0] = 0;
        set_error("moco_nce_step: bad enqueue argument (n_all=%d K=%d index=%lld)", n_all, K, (long long)index);
        return MOCO_ERR_INVALID;
    }
    const EnqueueSpec enq = {queue_bf16, queue_f32, k_all, k_all_dtype, n_all, (long long)index,
                             reinterpret_cast<long long*>(index_dev)};
    return nce_head(q, k, qk_dtype, normalize ? 1 : 0, queue_bf16, N, C, K, inv_T, nullptr, lse, loss_rows, prob_rows,
                    loss_prob, dq, workspace, workspace_bytes, flags, enq, static_cast<cudaStream_t>(stream_),
                    "moco_nce_step");
}

int moco_prof_sweep_window(const void* workspace, int n_ctas, float* us_out, void* stream_) {
    g_err[0] = 0;
    if (!workspace || !us_out || n_ctas < 1 || n_ctas > kMaxCtas) { set_error("moco_prof_sweep_window: bad argument"); return MOCO_ERR_INVALID; }
    NceWorkspace ws = carve_workspace(const_cast<void*>(workspace), 1, 64);
    static unsigned long long host[kMaxCtas * 2];
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    cudaError_t e = cudaMemcpyAsync(host, ws.cta_times, (size_t)n_ctas * 16, cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) return cuda_fail("moco_prof_sweep_window", e);
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
    if (kernel < 0 || kernel > 2) { set_error("moco_prof_set_events: bad kernel id"); return MOCO_ERR_INVALID; }
    g_prof_ev[kernel][0] = static_cast<cudaEvent_t>(ev_start);
    g_prof_ev[kernel][1] = static_cast<cudaEvent_t>(ev_stop);
    return MOCO_OK;
}

int moco_nce_bwd_dense(const float* grad_logits, const void* k, int k_dtype, const void* queue_bf16, int N, int C,
                       int K, float inv_T, float* dq, void* stream_) {
    g_err[0] = 0;
    if (!grad_logits || !k || !queue_bf16 || !dq || N <= 0 || C <= 0 || K <= 0) {
        set_error("moco_nce_bwd_dense: bad argument");
        return MOCO_ERR_INVALID;
    }
    cudaError_t e = launch_bwd_dense(grad_logits, k, k_dtype, static_cast<const __nv_bfloat16*>(queue_bf16), N, C, K,
                                     inv_T, dq, static_cast<cudaStream_t>(stream_));
    if (e != cudaSuccess) return cuda_fail("dense backward kernel", e);
    return MOCO_OK;
}

int moco_queue_enqueue(void* queue_bf16, float* queue_f32, const void* k_all, int k_dtype, int n_all, int C,
                       int64_t K, int64_t index, void* stream_) {
    g_err[0] = 0;
    if (!queue_bf16 || !k_all || n_all < 0 || C <= 0 || K <= 0 || index < 0 || index >= K) {
        set_error("moco_queue_enqueue: bad argument (n_all=%d C=%d K=%lld index=%lld)", n_all, C, (long long)K, (long long)index);
        return MOCO_ERR_INVALID;
    }
    if (n_all > K) {
        set_error("moco_queue_enqueue: n_all (%d) > K (%lld): write order would be ambiguous", n_all, (long long)K);
        return MOCO_ERR_INVALID;
    }
    cudaError_t e = launch_enqueue(static_cast<__nv_bfloat16*>(queue_bf16), queue_f32, k_all, k_dtype, n_all, C, K,
                                   index, 0, K, static_cast<cudaStream_t>(stream_));
    if (e != cudaSuccess) return cuda_fail("enqueue kernel", e);
    return MOCO_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Sharded queue (BASELINE configs[3]): every rank holds rows [shard_row0, shard_row0 + shard_rows) of the ring
// ---------------------------------------------------------------------------------------------------------
int moco_queue_enqueue_shard(void* shard_bf16, float* shard_f32, const void* k_all, int k_dtype, int n_all, int C,
                             int64_t K, int64_t index, int64_t shard_row0, int64_t shard_rows, void* stream_) {
    g_err[0] = 0;
    if (!shard_bf16 || !k_all || n_all < 0 || C <= 0 || K <= 0 || index < 0 || index >= K || n_all > K ||
        shard_row0 < 0 || shard_rows <= 0 || shard_row0 + shard_rows > K) {
        set_error("moco_queue_enqueue_shard: bad argument");
        return MOCO_ERR_INVALID;
    }
    cudaError_t e = launch_enqueue(static_cast<__nv_bfloat16*>(shard_bf16), shard_f32, k_all, k_dtype, n_all, C, K,
                                   index, shard_row0, shard_rows, static_cast<cudaStream_t>(stream_));
    if (e != cudaSuccess) return cuda_fail("enqueue kernel", e);
    return MOCO_OK;
}

static int shard_common(const char* what, const void* q, int N, int C, int Ks, void* workspace, size_t bytes,
                        NceWorkspace* ws, DevInfo* d) {
    if (!q || !workspace || N <= 0 || C <= 0 || Ks <= 0 || (reinterpret_cast<uintptr_t>(workspace) & 255)) {
        set_error("%s: bad argument", what);
        return MOCO_ERR_INVALID;
    }
    *ws = carve_workspace(workspace, N, C);
    if (bytes < ws->bytes) { set_error("%s: workspace too small (%zu < %zu)", what, bytes, ws->bytes); return MOCO_ERR_WORKSPACE; }
    *d = device_info();
    if (!d->ok || d->major != 9 || C % 64 != 0 || C > 256) {
        set_error("%s: needs an sm_90 device and C %% 64 == 0, C <= 256 (C=%d)", what, C);
        return MOCO_ERR_UNSUPPORTED;
    }
    return MOCO_OK;
}

int moco_nce_shard_stats(const void* q_all, const void* k_all, int qk_dtype, const void* shard_bf16, int N, int C,
                         int Ks, float inv_T, void* ms_out, void* workspace, size_t workspace_bytes, int flags,
                         void* stream_) {
    g_err[0] = 0;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    NceWorkspace ws; DevInfo d;
    int rc = shard_common("moco_nce_shard_stats", q_all, N, C, Ks, workspace, workspace_bytes, &ws, &d);
    if (rc != MOCO_OK) return rc;
    if (!k_all || !shard_bf16 || !ms_out) { set_error("moco_nce_shard_stats: null pointer"); return MOCO_ERR_INVALID; }
    cudaError_t e = launch_prep(q_all, k_all, qk_dtype, N, C, ws, stream);
    if (e != cudaSuccess) return cuda_fail("prep kernel", e);
    NceTcParams p;
    p.q_bf16 = qk_dtype == MOCO_BF16 ? static_cast<const __nv_bfloat16*>(q_all) : ws.q_bf16;
    p.queue = static_cast<const __nv_bfloat16*>(shard_bf16);
    p.N = N; p.C = C; p.K = Ks; p.inv_T = inv_T; p.logits = nullptr;
    p.cta_group = (flags & MOCO_NCE_CTA_PAIR) ? 2 : 1;
    p.num_sms = d.sms;
    p.slices = 0; p.n_pad = 0;
    if (flags & MOCO_NCE_ONE_PASS) {
        // one sweep over the shard: (stabiliser, sum) partials for the cross-rank merge AND the unnormalised
        // P~.Queue partials, which stay in the workspace until moco_nce_shard_dq(..., MOCO_NCE_ONE_PASS) rescales them
        e = launch_sweep(q_all, qk_dtype, 0, p.q_bf16, p.queue, N, C, Ks, inv_T, nullptr, d.sms, &p.slices, &p.n_pad, ws, stream);
        if (e != cudaSuccess) return cuda_fail("one-pass kernel", e);
    } else {
        e = launch_nce_tc(p, ws, stream);
        if (e != cudaSuccess) return cuda_fail("statistics kernel", e);
    }
    e = launch_combine_partial(N, p.slices, p.n_pad, static_cast<float2*>(ms_out), ws, stream);
    if (e != cudaSuccess) return cuda_fail("combine kernel", e);
    return MOCO_OK;
}

int moco_nce_shard_merge(const void* ms_all, int world, int N, int C, float inv_T, float* lse, float* loss_rows,
                         float* prob_rows, float* loss_prob, void* workspace, size_t workspace_bytes, void* stream_) {
    g_err[0] = 0;
    if (!ms_all || !lse || !loss_rows || !prob_rows || !loss_prob || !workspace || world < 1 || world > kMaxCtas || N <= 0) {
        set_error("moco_nce_shard_merge: bad argument");
        return MOCO_ERR_INVALID;
    }
    NceWorkspace ws = carve_workspace(workspace, N, C);
    if (workspace_bytes < ws.bytes) { set_error("moco_nce_shard_merge: workspace too small"); return MOCO_ERR_WORKSPACE; }
    cudaError_t e = launch_combine_merge(N, world, inv_T, static_cast<const float2*>(ms_all), lse, loss_rows, prob_rows,
                                         loss_prob, ws, static_cast<cudaStream_t>(stream_));
    if (e != cudaSuccess) return cuda_fail("combine kernel", e);
    return MOCO_OK;
}

int moco_nce_shard_dq(const void* q_all, int q_dtype, const void* shard_bf16, const float* lse_all, int N, int C,
                      int Ks, float inv_T, float* o_partial, void* workspace, size_t workspace_bytes, int flags,
                      void* stream_) {
    g_err[0] = 0;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    NceWorkspace ws; DevInfo d;
    int rc = shard_common("moco_nce_shard_dq", q_all, N, C, Ks, workspace, workspace_bytes, &ws, &d);
    if (rc != MOCO_OK) return rc;
    if (!shard_bf16 || !lse_all || !o_partial) { set_error("moco_nce_shard_dq: null pointer"); return MOCO_ERR_INVALID; }
    // q_bf16 in the workspace was produced by moco_nce_shard_stats on the same workspace (fp32 inputs)
    const __nv_bfloat16* qb = q_dtype == MOCO_BF16 ? static_cast<const __nv_bfloat16*>(q_all) : ws.q_bf16;
    int slices = 0, n_pad = 0;
    cudaError_t e;
    if (flags & MOCO_NCE_ONE_PASS) {
        // the sweep already happened in moco_nce_shard_stats(..., MOCO_NCE_ONE_PASS) on this workspace: only the
        // slice count is needed, then O = sum_s 2^(m_s - lse) O~_s
        e = launch_sweep(q_all, q_dtype, 0, qb, static_cast<const __nv_bfloat16*>(shard_bf16), N, C, Ks, inv_T, nullptr, d.sms,
                         &slices, &n_pad, ws, stream, /*plan_only=*/true);
        if (e != cudaSuccess) return cuda_fail("one-pass plan", e);
        e = launch_dq_reduce(N, C, slices, n_pad, inv_T, nullptr, 0, nullptr, o_partial, ws.part_o, stream, ws.part_ms, lse_all);
        if (e != cudaSuccess) return cuda_fail("dq reduce kernel", e);
        return MOCO_OK;
    }
    e = launch_sweep(q_all, q_dtype, 0, qb, static_cast<const __nv_bfloat16*>(shard_bf16), N, C, Ks, inv_T, lse_all, d.sms, &slices,
                     &n_pad, ws, stream);
    if (e != cudaSuccess) return cuda_fail("dq kernel", e);
    e = launch_dq_reduce(N, C, slices, n_pad, inv_T, nullptr, 0, nullptr, o_partial, ws.part_o, stream);
    if (e != cudaSuccess) return cuda_fail("dq reduce kernel", e);
    return MOCO_OK;
}

int moco_nce_shard_dq_finish(const float* o_own, const void* k_own, int k_dtype, const float* prob_rows_own, int N,
                             int C, float inv_T, float* dq, void* stream_) {
    g_err[0] = 0;
    if (!o_own || !k_own || !prob_rows_own || !dq || N <= 0 || C <= 0) {
        set_error("moco_nce_shard_dq_finish: bad argument");
        return MOCO_ERR_INVALID;
    }
    cudaError_t e = launch_dq_reduce(N, C, 1, N, inv_T, k_own, k_dtype, prob_rows_own, dq, o_own,
                                     static_cast<cudaStream_t>(stream_));
    if (e != cudaSuccess) return cuda_fail("dq finish kernel", e);
    return MOCO_OK;
}

int moco_nce_shard_dq_finish_peers(const void* const* o_peers_host, int world, int rank, const void* k_own, int k_dtype,
                                   const float* prob_rows_own, int N, int C, float inv_T, float* dq, void* stream_) {
    g_err[0] = 0;
    if (!o_peers_host || !k_own || !prob_rows_own || !dq || N <= 0 || C <= 0 || (C & 3) || world < 1 || world > 16 ||
        rank < 0 || rank >= world) {
        set_error("moco_nce_shard_dq_finish_peers: bad argument");
        return MOCO_ERR_INVALID;
    }
    for (int r = 0; r < world; ++r)
        if (!o_peers_host[r] || (reinterpret_cast<uintptr_t>(o_peers_host[r]) & 15)) {
            set_error("moco_nce_shard_dq_finish_peers: peer %d pointer null or misaligned", r);
            return MOCO_ERR_INVALID;
        }
    cudaError_t e = launch_dq_finish_peers(o_peers_host, world, rank, N, C, inv_T, k_own, k_dtype, prob_rows_own, dq,
                                           static_cast<cudaStream_t>(stream_));
    if (e != cudaSuccess) return cuda_fail("dq finish (peers) kernel", e);
    return MOCO_OK;
}

int moco_f32_to_bf16(const float* src, void* dst, size_t n, void* stream_) {
    g_err[0] = 0;
    if ((!src || !dst) && n) { set_error("moco_f32_to_bf16: null pointer"); return MOCO_ERR_INVALID; }
    cudaError_t e = launch_f32_to_bf16(src, static_cast<__nv_bfloat16*>(dst), n, static_cast<cudaStream_t>(stream_));
    if (e != cudaSuccess) return cuda_fail("f32->bf16 kernel", e);
    return MOCO_OK;
}

int moco_ema_chunk_elems(void) { return ema_chunk_elems(); }

int moco_ema_update(const void* segs, const int32_t* chunk_prefix, int n_segs, int n_chunks, float m, float one_minus_m,
                    void* stream_) {
    g_err[0] = 0;
    if (n_segs < 0 || n_chunks < 0 || ((!segs || !chunk_prefix) && n_segs > 0)) {
        set_error("moco_ema_update: bad argument");
        return MOCO_ERR_INVALID;
    }
    cudaError_t e = launch_ema(segs, chunk_prefix, n_segs, n_chunks, m, one_minus_m, static_cast<cudaStream_t>(stream_));
    if (e != cudaSuccess) return cuda_fail("ema kernel", e);
    return MOCO_OK;
}

int moco_crop_s2d_bf16(const void* src, int src_dtype, long long src_image_stride, const int64_t* src_rows, void* dst, int N,
                       int H, int W, void* stream_) {
    g_err[0] = 0;
    if (N < 0 || !dst || (!src && N) || (src_dtype != MOCO_F32 && src_dtype != MOCO_BF16) || src_image_stride < 3LL * H * W ||
        (reinterpret_cast<uintptr_t>(src) & 7) != 0 || (reinterpret_cast<uintptr_t>(dst) & 15) != 0 || (src_image_stride & 1) != 0) {
        set_error("moco_crop_s2d_bf16: bad argument");
        return MOCO_ERR_INVALID;
    }
    cudaError_t e = launch_crop_to_s2d(src, src_dtype, src_image_stride, static_cast<__nv_bfloat16*>(dst), N, H, W,
                                       static_cast<cudaStream_t>(stream_), src_rows);
    if (e == cudaErrorNotSupported) { set_error("moco_crop_s2d_bf16: needs even H, W >= 2 (H=%d W=%d)", H, W); return MOCO_ERR_UNSUPPORTED; }
    if (e != cudaSuccess) return cuda_fail("crop->space-to-depth kernel", e);
    return MOCO_OK;
}

int moco_maxpool3x3s2_fwd(const void* x, void* y, void* taps, int N, int H, int W, int C, void* stream_) {
    g_err[0] = 0;
    if (!x || !y || !taps || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 15) ||
        (reinterpret_cast<uintptr_t>(taps) & 7)) {
        set_error("moco_maxpool3x3s2_fwd: null or misaligned pointer");
        return MOCO_ERR_INVALID;
    }
    cudaError_t e = launch_maxpool_fwd(x, y, taps, N, H, W, C, static_cast<cudaStream_t>(stream_));
    if (e == cudaErrorNotSupported) { set_error("moco_maxpool3x3s2_fwd: needs N, H, W >= 1 and C %% 8 == 0 (C=%d)", C); return MOCO_ERR_UNSUPPORTED; }
    if (e != cudaSuccess) return cuda_fail("max-pool forward kernel", e);
    return MOCO_OK;
}

int moco_maxpool3x3s2_bwd(const void* dy, const void* taps, void* dx, int N, int H, int W, int C, void* stream_) {
    g_err[0] = 0;
    if (!dy || !dx || !taps || (reinterpret_cast<uintptr_t>(dy) & 15) || (reinterpret_cast<uintptr_t>(dx) & 15) ||
        (reinterpret_cast<uintptr_t>(taps) & 7)) {
        set_error("moco_maxpool3x3s2_bwd: null or misaligned pointer");
        return MOCO_ERR_INVALID;
    }
    cudaError_t e = launch_maxpool_bwd(dy, taps, dx, N, H, W, C, static_cast<cudaStream_t>(stream_));
    if (e == cudaErrorNotSupported) { set_error("moco_maxpool3x3s2_bwd: needs N, H, W >= 1 and C %% 8 == 0 (C=%d)", C); return MOCO_ERR_UNSUPPORTED; }
    if (e != cudaSuccess) return cuda_fail("max-pool backward kernel", e);
    return MOCO_OK;
}

size_t moco_bn_workspace_bytes(void) { return bn_workspace_bytes(); }

static bool misaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

int moco_bn_fwd_train(const void* x, const void* residual, void* y, long long M, int C, const float* gamma,
                      const float* beta, float* running_mean, float* running_var, long long* num_batches_tracked,
                      float momentum, float eps, int relu, float* save_mean, float* save_invstd, void* workspace,
                      size_t workspace_bytes, void* stream_) {
    g_err[0] = 0;
    if (!x || !y || !gamma || !beta || !save_mean || !save_invstd || !workspace || (running_mean == nullptr) != (running_var == nullptr) ||
        misaligned16(x) || misaligned16(y) || misaligned16(residual) || misaligned16(workspace) || x == y || !(eps > 0.f)) {
        set_error("moco_bn_fwd_train: bad argument (null / misaligned pointer, in-place, eps <= 0)");
        return MOCO_ERR_INVALID;
    }
    if (workspace_bytes < bn_workspace_bytes()) { set_error("moco_bn_fwd_train: workspace too small"); return MOCO_ERR_WORKSPACE; }
    cudaError_t e = launch_bn_fwd_train(x, residual, y, M, C, gamma, beta, running_mean, running_var, num_batches_tracked,
                                        momentum, eps, relu, save_mean, save_invstd, workspace, static_cast<cudaStream_t>(stream_));
    if (e == cudaErrorNotSupported) {
        set_error("moco_bn_fwd_train: needs M >= 1 and C a power of two in [64, 2048] (M=%lld C=%d)", M, C);
        return MOCO_ERR_UNSUPPORTED;
    }
    if (e != cudaSuccess) return cuda_fail("batch-norm forward kernels", e);
    return MOCO_OK;
}

int moco_bn_bwd(const void* dy, const void* x, const void* y, long long M, int C, const float* gamma, const float* beta,
                const float* save_mean, const float* save_invstd, int relu, int has_residual, void* dx, void* dresidual,
                float* dgamma, float* dbeta, void* workspace, size_t workspace_bytes, void* stream_) {
    g_err[0] = 0;
    if (!dy || !x || !dx || !gamma || !beta || !save_mean || !save_invstd || !dgamma || !dbeta || !workspace ||
        (relu && has_residual && !y) || misaligned16(dy) || misaligned16(x) || misaligned16(y) || misaligned16(dx) ||
        misaligned16(dresidual) || misaligned16(workspace)) {
        set_error("moco_bn_bwd: bad argument (null / misaligned pointer; y is required with relu + residual)");
        return MOCO_ERR_INVALID;
    }
    if (workspace_bytes < bn_workspace_bytes()) { set_error("moco_bn_bwd: workspace too small"); return MOCO_ERR_WORKSPACE; }
    cudaError_t e = launch_bn_bwd(dy, x, y, M, C, gamma, beta, save_mean, save_invstd, relu, has_residual, dx, dresidual,
                                  dgamma, dbeta, workspace, static_cast<cudaStream_t>(stream_));
    if (e == cudaErrorNotSupported) {
        set_error("moco_bn_bwd: needs M >= 1 and C a power of two in [64, 2048] (M=%lld C=%d)", M, C);
        return MOCO_ERR_UNSUPPORTED;
    }
    if (e != cudaSuccess) return cuda_fail("batch-norm backward kernels", e);
    return MOCO_OK;
}

static bool bn_layer_fwd_ok(const moco_bn_layer* b) {
    return b && b->gamma && b->beta && b->save_mean && b->save_invstd &&
           (b->running_mean == nullptr) == (b->running_var == nullptr) && b->eps > 0.f;
}

static bool bn_layer_bwd_ok(const moco_bn_layer* b) {
    return b && b->gamma && b->save_mean && b->save_invstd && b->dgamma && b->dbeta;
}

int moco_bn_add_relu_fwd_train(const void* x, const void* residual, void* y, void* mask, long long M, int C,
                               const moco_bn_layer* bn, const moco_bn_layer* shortcut, void* workspace,
                               size_t workspace_bytes, void* stream_) {
    g_err[0] = 0;
    if (!x || !residual || !y || !workspace || !bn_layer_fwd_ok(bn) || (shortcut && !bn_layer_fwd_ok(shortcut)) ||
        misaligned16(x) || misaligned16(residual) || misaligned16(y) || misaligned16(workspace) || x == y || residual == y) {
        set_error("moco_bn_add_relu_fwd_train: bad argument (null / misaligned pointer, in-place, eps <= 0, "
                  "one of running_mean / running_var)");
        return MOCO_ERR_INVALID;
    }
    if (workspace_bytes < bn_workspace_bytes()) { set_error("moco_bn_add_relu_fwd_train: workspace too small"); return MOCO_ERR_WORKSPACE; }
    cudaError_t e = launch_bn_add_relu_fwd(x, residual, y, mask, M, C, *bn, shortcut, workspace,
                                           static_cast<cudaStream_t>(stream_));
    if (e == cudaErrorNotSupported) {
        set_error("moco_bn_add_relu_fwd_train: needs M >= 1 and C a power of two in [64, 2048] (M=%lld C=%d)", M, C);
        return MOCO_ERR_UNSUPPORTED;
    }
    if (e != cudaSuccess) return cuda_fail("batch-norm forward kernels", e);
    return MOCO_OK;
}

int moco_bn_add_relu_bwd(const void* dy, const void* x, const void* residual, const void* mask, long long M, int C,
                         const moco_bn_layer* bn, const moco_bn_layer* shortcut, void* dx, void* dresidual,
                         void* workspace, size_t workspace_bytes, void* stream_) {
    g_err[0] = 0;
    if (!dy || !x || !mask || !dx || !workspace || !bn_layer_bwd_ok(bn) ||
        (shortcut && (!bn_layer_bwd_ok(shortcut) || !residual || !dresidual)) || misaligned16(dy) || misaligned16(x) ||
        misaligned16(residual) || misaligned16(dx) || misaligned16(dresidual) || misaligned16(workspace)) {
        set_error("moco_bn_add_relu_bwd: bad argument (null / misaligned pointer; residual and dresidual are required "
                  "with a shortcut BN)");
        return MOCO_ERR_INVALID;
    }
    if (workspace_bytes < bn_workspace_bytes()) { set_error("moco_bn_add_relu_bwd: workspace too small"); return MOCO_ERR_WORKSPACE; }
    cudaError_t e = launch_bn_add_relu_bwd(dy, x, residual, mask, M, C, *bn, shortcut, dx, dresidual, workspace,
                                           static_cast<cudaStream_t>(stream_));
    if (e == cudaErrorNotSupported) {
        set_error("moco_bn_add_relu_bwd: needs M >= 1 and C a power of two in [64, 2048] (M=%lld C=%d)", M, C);
        return MOCO_ERR_UNSUPPORTED;
    }
    if (e != cudaSuccess) return cuda_fail("batch-norm backward kernels", e);
    return MOCO_OK;
}

int moco_bn_relu_maxpool_fwd_train(const void* x, void* y, void* taps, int N, int H, int W, int C,
                                   const moco_bn_layer* bn, void* workspace, size_t workspace_bytes, void* stream_) {
    g_err[0] = 0;
    if (!x || !y || !taps || !workspace || !bn_layer_fwd_ok(bn) || misaligned16(x) || misaligned16(y) ||
        (reinterpret_cast<uintptr_t>(taps) & 7) || misaligned16(workspace)) {
        set_error("moco_bn_relu_maxpool_fwd_train: bad argument (null / misaligned pointer, eps <= 0, "
                  "one of running_mean / running_var)");
        return MOCO_ERR_INVALID;
    }
    if (workspace_bytes < bn_workspace_bytes()) { set_error("moco_bn_relu_maxpool_fwd_train: workspace too small"); return MOCO_ERR_WORKSPACE; }
    cudaError_t e = launch_bn_relu_maxpool_fwd(x, y, taps, N, H, W, C, *bn, workspace, static_cast<cudaStream_t>(stream_));
    if (e == cudaErrorNotSupported) {
        set_error("moco_bn_relu_maxpool_fwd_train: needs N, H, W >= 1 and C a power of two in [64, 2048] (C=%d)", C);
        return MOCO_ERR_UNSUPPORTED;
    }
    if (e != cudaSuccess) return cuda_fail("batch-norm + max-pool forward kernels", e);
    return MOCO_OK;
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
    if (!x || !y || !bn_eval_coefs_ok(scale, shift, residual, sc_scale, sc_shift) || misaligned16(x) ||
        misaligned16(residual) || misaligned16(y) || x == y || residual == y) {
        set_error("moco_bn_eval_act: bad argument (null / misaligned pointer, in-place, one of sc_scale / sc_shift, "
                  "a shortcut BN without a residual)");
        return MOCO_ERR_INVALID;
    }
    cudaError_t e = launch_bn_eval_act(x, residual, y, M, C, scale, shift, relu, sc_scale, sc_shift,
                                       static_cast<cudaStream_t>(stream_));
    if (e == cudaErrorNotSupported) {
        set_error("moco_bn_eval_act: needs M >= 1 and C a power of two in [64, 2048] (M=%lld C=%d)", M, C);
        return MOCO_ERR_UNSUPPORTED;
    }
    if (e != cudaSuccess) return cuda_fail("batch-norm eval kernel", e);
    return MOCO_OK;
}

int moco_bn_relu_maxpool_eval(const void* x, void* y, int N, int H, int W, int C, const float* scale,
                              const float* shift, void* stream_) {
    g_err[0] = 0;
    if (!x || !y || !scale || !shift || misaligned16(x) || misaligned16(y) || x == y) {
        set_error("moco_bn_relu_maxpool_eval: bad argument (null / misaligned pointer, in-place)");
        return MOCO_ERR_INVALID;
    }
    cudaError_t e = launch_bn_relu_maxpool_eval(x, y, N, H, W, C, scale, shift, static_cast<cudaStream_t>(stream_));
    if (e == cudaErrorNotSupported) {
        set_error("moco_bn_relu_maxpool_eval: needs N, H, W >= 1 and C a power of two in [64, 2048] (C=%d)", C);
        return MOCO_ERR_UNSUPPORTED;
    }
    if (e != cudaSuccess) return cuda_fail("batch-norm eval + max-pool kernel", e);
    return MOCO_OK;
}

int moco_bn_eval_act_avgpool(const void* x, const void* residual, float* feat, int N, int HW, int C, const float* scale,
                             const float* shift, int relu, const float* sc_scale, const float* sc_shift, void* stream_) {
    g_err[0] = 0;
    if (!x || !feat || !bn_eval_coefs_ok(scale, shift, residual, sc_scale, sc_shift) || misaligned16(x) ||
        misaligned16(residual) || misaligned16(feat)) {
        set_error("moco_bn_eval_act_avgpool: bad argument (null / misaligned pointer, one of sc_scale / sc_shift, "
                  "a shortcut BN without a residual)");
        return MOCO_ERR_INVALID;
    }
    cudaError_t e = launch_bn_eval_act_avgpool(x, residual, feat, N, HW, C, scale, shift, relu, sc_scale, sc_shift,
                                               static_cast<cudaStream_t>(stream_));
    if (e == cudaErrorNotSupported) {
        set_error("moco_bn_eval_act_avgpool: needs N, HW >= 1 and C a power of two in [64, 2048] (N=%d HW=%d C=%d)", N,
                  HW, C);
        return MOCO_ERR_UNSUPPORTED;
    }
    if (e != cudaSuccess) return cuda_fail("batch-norm eval + average-pool kernel", e);
    return MOCO_OK;
}

int moco_crop_to_nhwc_bf16(const void* src, int src_dtype, long long src_image_stride, void* dst, int N, int C, int HW,
                           void* stream_) {
    g_err[0] = 0;
    if (N < 0 || !dst || (!src && N) || (src_dtype != MOCO_F32 && src_dtype != MOCO_BF16) || src_image_stride < (long long)C * HW ||
        (reinterpret_cast<uintptr_t>(src) & 15) != 0 || (reinterpret_cast<uintptr_t>(dst) & 15) != 0 ||
        (src_image_stride & (src_dtype == MOCO_F32 ? 3 : 7)) != 0) {
        set_error("moco_crop_to_nhwc_bf16: bad argument");
        return MOCO_ERR_INVALID;
    }
    cudaError_t e = launch_crop_to_nhwc(src, src_dtype, src_image_stride, static_cast<__nv_bfloat16*>(dst), N, C, HW,
                                        static_cast<cudaStream_t>(stream_));
    if (e == cudaErrorNotSupported) { set_error("moco_crop_to_nhwc_bf16: needs C <= 4 and H*W %% 8 == 0 (C=%d HW=%d)", C, HW); return MOCO_ERR_UNSUPPORTED; }
    if (e != cudaSuccess) return cuda_fail("crop->nhwc kernel", e);
    return MOCO_OK;
}

static int shuffle_gather_impl(const void* const* peers, int world, int rows_per_rank, const int64_t* src_rows, int n_rows,
                               size_t row_bytes, void* dst, int flags, void* stream_, void* const* pads, int rank,
                               uint32_t epoch);

int moco_shuffle_gather(const void* const* peers, int world, int rows_per_rank, const int64_t* src_rows, int n_rows,
                        size_t row_bytes, void* dst, int flags, void* stream_) {
    return shuffle_gather_impl(peers, world, rows_per_rank, src_rows, n_rows, row_bytes, dst, flags, stream_, nullptr, 0, 0);
}

int moco_shuffle_gather_sync(const void* const* peers, void* const* pads, int world, int rank, uint32_t epoch,
                             int rows_per_rank, const int64_t* src_rows, int n_rows, size_t row_bytes, void* dst,
                             int flags, void* stream_) {
    if (!pads || rank < 0 || rank >= world || epoch == 0) {
        g_err[0] = 0;
        set_error("moco_shuffle_gather_sync: bad synchronisation argument (rank=%d world=%d epoch=%u)", rank, world, epoch);
        return MOCO_ERR_INVALID;
    }
    return shuffle_gather_impl(peers, world, rows_per_rank, src_rows, n_rows, row_bytes, dst, flags, stream_, pads, rank, epoch);
}

int moco_p2p_last_timeout(uint32_t out[4]) {
    g_err[0] = 0;
    unsigned int* w = p2p_status_words();
    if (!out || !w) { set_error("moco_p2p_last_timeout: no status block"); return MOCO_ERR_INVALID; }
    for (int i = 0; i < 4; ++i) out[i] = w[i];
    return MOCO_OK;
}

int moco_crop_gather_nhwc_bf16(const void* src, int src_dtype, long long src_image_stride, const int64_t* src_rows,
                               void* dst, int N, int C, int HW, void* stream_) {
    g_err[0] = 0;
    if (N < 0 || !dst || (!src && N) || (src_dtype != MOCO_F32 && src_dtype != MOCO_BF16) || src_image_stride < (long long)C * HW ||
        (reinterpret_cast<uintptr_t>(src) & 15) != 0 || (reinterpret_cast<uintptr_t>(dst) & 15) != 0 ||
        (src_image_stride & (src_dtype == MOCO_F32 ? 3 : 7)) != 0) {
        set_error("moco_crop_gather_nhwc_bf16: bad argument");
        return MOCO_ERR_INVALID;
    }
    cudaError_t e = launch_crop_to_nhwc(src, src_dtype, src_image_stride, static_cast<__nv_bfloat16*>(dst), N, C, HW,
                                        static_cast<cudaStream_t>(stream_), src_rows);
    if (e == cudaErrorNotSupported) { set_error("moco_crop_gather_nhwc_bf16: needs C <= 4 and H*W %% 8 == 0 (C=%d HW=%d)", C, HW); return MOCO_ERR_UNSUPPORTED; }
    if (e != cudaSuccess) return cuda_fail("crop->nhwc kernel", e);
    return MOCO_OK;
}

static int shuffle_gather_impl(const void* const* peers, int world, int rows_per_rank, const int64_t* src_rows, int n_rows,
                               size_t row_bytes, void* dst, int flags, void* stream_, void* const* pads, int rank,
                               uint32_t epoch) {
    g_err[0] = 0;
    if (!peers || !src_rows || !dst || world < 1 || world > 16 || rows_per_rank < 1 || n_rows < 0 ||
        row_bytes == 0 || (row_bytes & 15) != 0 || (reinterpret_cast<uintptr_t>(dst) & 15) != 0) {
        set_error("moco_shuffle_gather: bad argument (world=%d rows_per_rank=%d n_rows=%d row_bytes=%zu)", world,
                  rows_per_rank, n_rows, row_bytes);
        return MOCO_ERR_INVALID;
    }
    for (int i = 0; i < world; ++i)
        if (!peers[i] || (reinterpret_cast<uintptr_t>(peers[i]) & 15) != 0) {
            set_error("moco_shuffle_gather: peer %d pointer null or misaligned", i);
            return MOCO_ERR_INVALID;
        }
    cudaError_t e = launch_gather(peers, world, rows_per_rank, src_rows, n_rows, row_bytes, dst, flags,
                                  static_cast<cudaStream_t>(stream_), pads, rank, epoch);
    if (e != cudaSuccess) return cuda_fail("shuffle gather kernel", e);
    return MOCO_OK;
}

int moco_signal_barrier(void* const* pads, int world, int rank, uint32_t epoch, void* stream_) {
    g_err[0] = 0;
    if (!pads || world < 1 || world > 16 || rank < 0 || rank >= world) {
        set_error("moco_signal_barrier: bad argument");
        return MOCO_ERR_INVALID;
    }
    cudaError_t e = launch_signal_barrier(pads, world, rank, epoch, static_cast<cudaStream_t>(stream_));
    if (e != cudaSuccess) return cuda_fail("signal barrier kernel", e);
    return MOCO_OK;
}

int moco_p2p_alloc(size_t bytes, void** dev_ptr_out, unsigned char handle_out[64]) {
    g_err[0] = 0;
    if (!dev_ptr_out || !handle_out || bytes == 0) { set_error("moco_p2p_alloc: bad argument"); return MOCO_ERR_INVALID; }
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) return cuda_fail("cudaMalloc", e);
    e = cudaMemset(p, 0, bytes);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { cudaFree(p); return cuda_fail("cudaMemset", e); }
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    cudaIpcMemHandle_t h;
    e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) { cudaFree(p); return cuda_fail("cudaIpcGetMemHandle", e); }
    memcpy(handle_out, &h, 64);
    *dev_ptr_out = p;
    return MOCO_OK;
}

int moco_p2p_open(const unsigned char handle[64], void** dev_ptr_out) {
    g_err[0] = 0;
    if (!handle || !dev_ptr_out) { set_error("moco_p2p_open: bad argument"); return MOCO_ERR_INVALID; }
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    void* p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return cuda_fail("cudaIpcOpenMemHandle", e);
    *dev_ptr_out = p;
    return MOCO_OK;
}

int moco_p2p_close(void* dev_ptr) {
    g_err[0] = 0;
    cudaError_t e = cudaIpcCloseMemHandle(dev_ptr);
    if (e != cudaSuccess) return cuda_fail("cudaIpcCloseMemHandle", e);
    return MOCO_OK;
}

int moco_p2p_free(void* dev_ptr) {
    g_err[0] = 0;
    cudaError_t e = cudaFree(dev_ptr);
    if (e != cudaSuccess) return cuda_fail("cudaFree", e);
    return MOCO_OK;
}

}  // extern "C"
