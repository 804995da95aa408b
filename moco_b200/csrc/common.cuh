// Shared declarations for the moco_b200 CUDA sources.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>

#include "../../include/moco_b200.h"

namespace moco {

constexpr int kMaxCtas = 160;          // upper bound on persistent CTAs (H100 SXM: 132 SMs)
constexpr int kRowsPerCta = 128;       // q rows per CTA in the tensor-core kernels (two 64-row warpgroups)
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

// Workspace layout shared by every NCE entry point.
struct NceWorkspace {
    unsigned int* counters;   // [4]   (zeroed by the prep / sweep kernel each call)
    unsigned long long* cta_times;   // [kMaxCtas][2] %globaltimer at entry / exit of every CTA of the last sweep kernel
    float* lpos;              // [N]   <q_i, k_i> in fp32, natural units
    __nv_bfloat16* q_bf16;    // [N, C] bf16 copy of q (when q arrives as fp32)
    float2* part_ms;          // [slices, N_pad] per-slice (running max, sum) in the log2 domain
    float* part_o;            // [slices, N_pad, C] per-slice unnormalised sum_j 2^(x_ij - m) queue_j
    size_t bytes;
};

// Programmatic dependent launch for the head's kernel chain (prep -> one-pass | stats -> combine [-> dq] -> dq_reduce
// -> enqueue): at MoCo's default shape each of these kernels is a few microseconds, so grid launch latency and CTA
// start-up are a large share of the chain; PDL overlaps them with the predecessor's execution.  MOCO_PDL=0 turns
// the attribute off (A/B timing).  Only kernels that call pdl_wait() before their first global access use this.
inline bool pdl_enabled() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("MOCO_PDL"); v = (e && e[0] == '0') ? 0 : 1; }
    return v == 1;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

inline NceWorkspace carve_workspace(void* base, int N, int C) {
    NceWorkspace w;
    char* p = static_cast<char*>(base);
    size_t off = 0;
    w.counters = reinterpret_cast<unsigned int*>(p + off);            off += 256;
    w.cta_times = reinterpret_cast<unsigned long long*>(p + off);     off += align_up((size_t)kMaxCtas * 16, 256);
    w.lpos = reinterpret_cast<float*>(p + off);                       off += align_up((size_t)N * 4, 256);
    w.q_bf16 = reinterpret_cast<__nv_bfloat16*>(p + off);             off += align_up((size_t)N * C * 2, 256);
    w.part_ms = reinterpret_cast<float2*>(p + off);                   off += align_up((size_t)kMaxCtas * kRowsPerCta * 8, 256);
    w.part_o = reinterpret_cast<float*>(p + off);                     off += align_up((size_t)kMaxCtas * kRowsPerCta * C * 4, 256);
    w.bytes = off;
    return w;
}

// ---- launchers implemented across the .cu files (all async on `stream`) ----
cudaError_t launch_prep(const void* q, const void* k, int qk_dtype, int N, int C,
                        const NceWorkspace& ws, cudaStream_t stream);
cudaError_t launch_simt_rows(const __nv_bfloat16* q_bf16, const void* k, int k_dtype,
                             const __nv_bfloat16* queue, int N, int C, int K, float inv_T,
                             float* logits, float* lse, float* loss_rows, float* prob_rows,
                             float* loss_prob, float* dq, const NceWorkspace& ws, cudaStream_t stream);
cudaError_t launch_combine(int N, int C, int slices, int n_pad, float inv_T, float* logits, int K,
                           float* lse, float* loss_rows, float* prob_rows, float* loss_prob,
                           const NceWorkspace& ws, cudaStream_t stream);
cudaError_t launch_dq_reduce(int N, int C, int slices, int n_pad, float inv_T, const void* k, int k_dtype,
                             const float* prob_rows, float* dq, const float* part_o, cudaStream_t stream,
                             const float2* part_ms = nullptr, const float* lse = nullptr);
cudaError_t launch_dq_finish_peers(const void* const* peers_host, int world, int rank, int N, int C, float inv_T,
                                   const void* k, int k_dtype, const float* prob_rows, float* dq, cudaStream_t stream);
cudaError_t launch_combine_partial(int N, int slices, int n_pad, float2* ms_out, const NceWorkspace& ws,
                                   cudaStream_t stream);
cudaError_t launch_combine_merge(int N, int world, float inv_T, const float2* ms_all, float* lse, float* loss_rows,
                                 float* prob_rows, float* loss_prob, const NceWorkspace& ws, cudaStream_t stream);
cudaError_t launch_bwd_dense(const float* g, const void* k, int k_dtype, const __nv_bfloat16* queue,
                             int N, int C, int K, float inv_T, float* dq, cudaStream_t stream);
cudaError_t launch_enqueue(__nv_bfloat16* queue_bf16, float* queue_f32, const void* k_all, int k_dtype,
                           int n_all, int C, int64_t K, int64_t index, int64_t shard_row0, int64_t shard_rows,
                           cudaStream_t stream);
cudaError_t launch_f32_to_bf16(const float* src, __nv_bfloat16* dst, size_t n, cudaStream_t stream);
// bn_*: nullable; the stem's BatchNorm + ReLU applied to each tap (moco_bn_relu_maxpool_fwd_train).
// eval_scale / eval_shift: nullable; the same with a frozen BatchNorm's folded coefficients (moco_bn_relu_maxpool_eval),
// idx may then be NULL (no tap bytes are written).
cudaError_t launch_maxpool_fwd(const void* x, void* y, void* idx, int N, int H, int W, int C, cudaStream_t stream,
                               const float* bn_mean = nullptr, const float* bn_invstd = nullptr,
                               const float* bn_gamma = nullptr, const float* bn_beta = nullptr,
                               const float* eval_scale = nullptr, const float* eval_shift = nullptr);
cudaError_t launch_maxpool_bwd(const void* dy, const void* idx, void* dx, int N, int H, int W, int C, cudaStream_t stream);
cudaError_t launch_crop_to_s2d(const void* src, int src_dtype, long long img_stride, __nv_bfloat16* dst, int N, int H, int W,
                               cudaStream_t stream, const int64_t* src_rows);
size_t bn_workspace_bytes();
cudaError_t launch_bn_fwd_train(const void* x, const void* res, void* y, long long M, int C, const float* gamma,
                                const float* beta, float* running_mean, float* running_var, long long* nbt, float momentum,
                                float eps, int relu, float* save_mean, float* save_invstd, void* ws, cudaStream_t stream);
cudaError_t launch_bn_bwd(const void* dy, const void* x, const void* y, long long M, int C, const float* gamma,
                          const float* beta, const float* save_mean, const float* save_invstd, int relu, int has_residual,
                          void* dx, void* dres, float* dgamma, float* dbeta, void* ws, cudaStream_t stream);
using BnLayer = moco_bn_layer;
cudaError_t launch_bn_add_relu_fwd(const void* x, const void* res, void* y, void* mask, long long M, int C,
                                   const BnLayer& bn, const BnLayer* sc, void* ws, cudaStream_t stream);
cudaError_t launch_bn_add_relu_bwd(const void* dy, const void* x, const void* res, const void* mask, long long M, int C,
                                   const BnLayer& bn, const BnLayer* sc, void* dx, void* dres, void* ws,
                                   cudaStream_t stream);
cudaError_t launch_bn_relu_maxpool_fwd(const void* x, void* y, void* taps, int N, int H, int W, int C, const BnLayer& bn,
                                       void* ws, cudaStream_t stream);
cudaError_t launch_bn_eval_act(const void* x, const void* res, void* y, long long M, int C, const float* scale,
                               const float* shift, int relu, const float* sc_scale, const float* sc_shift,
                               cudaStream_t stream);
cudaError_t launch_bn_eval_act_avgpool(const void* x, const void* res, float* feat, int N, int HW, int C,
                                       const float* scale, const float* shift, int relu, const float* sc_scale,
                                       const float* sc_shift, cudaStream_t stream);
cudaError_t launch_bn_relu_maxpool_eval(const void* x, void* y, int N, int H, int W, int C, const float* scale,
                                        const float* shift, cudaStream_t stream);
int ema_chunk_elems();
cudaError_t launch_ema(const void* segs, const int* chunk_prefix, int n_segs, int n_chunks, float m,
                       float one_minus_m, cudaStream_t stream);
cudaError_t launch_crop_to_nhwc(const void* src, int src_dtype, long long img_stride, __nv_bfloat16* dst, int N, int C,
                                int HW, cudaStream_t stream, const int64_t* src_rows = nullptr);
cudaError_t launch_gather(const void* const* peers, int world, int rows_per_rank, const int64_t* src_rows,
                          int n_rows, size_t row_bytes, void* dst, int flags, cudaStream_t stream,
                          void* const* pads_host = nullptr, int rank = 0, uint32_t epoch = 0);
unsigned int* p2p_status_words();
cudaError_t launch_signal_barrier(void* const* pads, int world, int rank, uint32_t epoch, cudaStream_t stream);

// wgmma kernels (nce_sweep_sm90.cu).  Return cudaErrorNotSupported when the shape is not handled.
struct NceTcParams {
    const __nv_bfloat16* q_bf16;   // [N, C]
    const __nv_bfloat16* queue;    // [K, C]
    int N, C, K;
    float inv_T;
    float* logits;                 // optional dense [N, K+1]
    int cta_group;                 // 1, or 2: CTA pairs sharing every queue tile by TMA multicast
    int num_sms;
    // outputs of the launch decision
    int slices;
    int n_pad;
};
cudaError_t launch_nce_tc(NceTcParams& p, const NceWorkspace& ws, cudaStream_t stream);
// the q.Queue^T sweep with the gradient partials (one-sweep mode when lse == nullptr) and the fused tail (nce_tail.cu)
cudaError_t launch_nce_sweep(const void* q, int q_dtype, int normalize, const __nv_bfloat16* queue, int N, int C, int K,
                             float inv_T, const float* lse, int num_sms, int* slices_out, int* n_pad_out,
                             const NceWorkspace& ws, cudaStream_t stream, bool plan_only = false);
bool nce_tail_can_enqueue(int C, int normalize);
cudaError_t launch_nce_tail(int N, int C, int K, int slices, int n_pad, float inv_T, const void* q, const void* k,
                            int qk_dtype, int normalize, const __nv_bfloat16* queue, float* lse, float* loss_rows,
                            float* prob_rows, float* loss_prob, float* dq, const NceWorkspace& ws,
                            __nv_bfloat16* enq_bf16, float* enq_f32, const void* k_all, int k_all_dtype, int n_all,
                            long long index, long long* index_dev, long long row0, long long nrows, cudaStream_t stream);

void set_error(const char* fmt, ...);

}  // namespace moco
