// Shared declarations for the moco_b200 CUDA sources.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>

#include <atomic>

#include "../../include/moco_b200.h"

namespace moco {

constexpr int kMaxCtas = 160;          // upper bound on persistent CTAs (H100 SXM: 132 SMs)
constexpr int kRowsPerCta = 128;       // q rows per CTA in the tensor-core kernels (two 64-row warpgroups)
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

// Workspace layout shared by every NCE entry point.
struct NceWorkspace {
    unsigned int* counters;   // [4]   (zeroed by the prep / sweep kernel each call): [0] last-block means,
                              //       [1] the tail's enqueue release, [2] the separate enqueue's last block
    unsigned long long* cta_times;   // [kMaxCtas][2] %globaltimer at entry / exit of every CTA of the last sweep kernel
    float* lpos;              // [N]   <q_i, k_i> in fp32, natural units
    __nv_bfloat16* q_bf16;    // [N, C] bf16 copy of q (when q arrives as fp32)
    float2* part_ms;          // [slices, N_pad] per-slice (running max, sum) in the log2 domain
    float* part_o;            // [slices, N_pad, C] per-slice unnormalised sum_j 2^(x_ij - m) queue_j
    int* row_exact;           // [N]   sharded one-sweep mode: 1 where the statistics call evaluated the row exactly,
                              //       so the dq call must too (ShardExact below)
    size_t bytes;
};

// Exact CUDA-core evaluation of the rows the sharded one-sweep kernel cannot represent (moco_nce_shard_stats /
// moco_nce_shard_dq with MOCO_NCE_ONE_PASS).  row_exact == nullptr: no such evaluation (two-pass mode).
struct ShardExact {
    int* row_exact;                  // [N] per-row decision, written by the statistics call, read by the dq call
    const __nv_bfloat16* q;          // [N, C] bf16(q)
    const __nv_bfloat16* shard;      // [Ks, C]
    int Ks;
    float inv_T;
};

// The kernels launched in this process (moco_launch_count).  Every launch of the library passes its result through
// counted(): launch_pdl and launch_cluster wrap cudaLaunchKernelEx in it, and each <<<...>>> is followed by launched().
extern std::atomic<unsigned long long> g_launch_count;
inline cudaError_t counted(cudaError_t e) {
    if (e == cudaSuccess) g_launch_count.fetch_add(1, std::memory_order_relaxed);
    return e;
}
inline cudaError_t launched() { return counted(cudaGetLastError()); }

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
    return counted(cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...));
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
    w.row_exact = reinterpret_cast<int*>(p + off);                    off += align_up((size_t)N * 4, 256);
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
                             const float2* part_ms = nullptr, const float* lse = nullptr,
                             const ShardExact& exact = ShardExact{nullptr, nullptr, nullptr, 0, 0.f});
cudaError_t launch_dq_finish_peers(const void* const* peers_host, int world, int rank, int N, int C, float inv_T,
                                   const void* k, int k_dtype, const float* prob_rows, float* dq, cudaStream_t stream);
cudaError_t launch_combine_partial(int N, int C, int slices, int n_pad, float2* ms_out, const NceWorkspace& ws,
                                   const ShardExact& exact, cudaStream_t stream);
cudaError_t launch_combine_merge(int N, int world, float inv_T, const float2* ms_all, float* lse, float* loss_rows,
                                 float* prob_rows, float* loss_prob, const NceWorkspace& ws, cudaStream_t stream);
cudaError_t launch_bwd_dense(const float* g, const void* k, int k_dtype, const __nv_bfloat16* queue,
                             int N, int C, int K, float inv_T, float* dq, cudaStream_t stream);
// index_dev != nullptr: the ring position is read from and advanced on the device; `done` is a zeroed workspace
// counter the kernel uses to find its last block (and re-arms).
cudaError_t launch_enqueue(__nv_bfloat16* queue_bf16, float* queue_f32, const void* k_all, int k_dtype,
                           int n_all, int C, int64_t K, int64_t index, int64_t shard_row0, int64_t shard_rows,
                           cudaStream_t stream, long long* index_dev = nullptr, unsigned int* done = nullptr);
cudaError_t launch_f32_to_bf16(const float* src, __nv_bfloat16* dst, size_t n, cudaStream_t stream);
// bn_*: nullable; the stem's BatchNorm + ReLU applied to each tap (moco_bn_relu_maxpool_fwd_train).
// eval_scale / eval_shift: nullable; the same with a frozen BatchNorm's folded coefficients (moco_bn_relu_maxpool_eval),
// idx may then be NULL (no tap bytes are written).
cudaError_t launch_maxpool_fwd(const void* x, void* y, void* idx, int N, int H, int W, int C, cudaStream_t stream,
                               const float* bn_mean = nullptr, const float* bn_invstd = nullptr,
                               const float* bn_gamma = nullptr, const float* bn_beta = nullptr,
                               const float* eval_scale = nullptr, const float* eval_shift = nullptr);
// dy2: nullable; a second gradient of the pooled output, added to dy (bf16 rounding of the sum) before the gather
cudaError_t launch_maxpool_bwd(const void* dy, const void* dy2, const void* idx, void* dx, int N, int H, int W, int C,
                               cudaStream_t stream);
cudaError_t launch_crop_to_s2d(const void* src, int src_dtype, long long img_stride, __nv_bfloat16* dst, int N, int H, int W,
                               cudaStream_t stream, const int64_t* src_rows);
size_t bn_workspace_bytes();
using BnLayer = moco_bn_layer;
// a BatchNorm reduction's workspace: the slabs' ticket counters (zero between calls) at ws, then the per-CTA partials
inline float* bn_ws_partials(void* ws) { return reinterpret_cast<float*>(static_cast<char*>(ws) + 256); }
struct BnFwdPlan {              // the training forward: launch_bn_stats of each layer not `given`, then one apply pass
    const void *x, *res;           // res: nullable; with sc the shortcut BN's input, added as bf16(sc(res))
    void *y, *mask, *ws;           // mask: nullable, the ReLU mask bits of y for the backward; ws: unless all are given
    const BnLayer *bn, *sc;        // sc: nullable, a downsample block's shortcut BN
    long long M;
    int C, relu, given;            // given: MOCO_BN_STATS_GIVEN | MOCO_BN_SC_STATS_GIVEN, whose save_* are final
};
cudaError_t launch_bn_fwd(const BnFwdPlan& f, cudaStream_t stream);
struct BnBwdPlan {              // the training backward: the reduction pass (dbeta, dgamma), then the element-wise pass
    const void *dy, *dy2, *x;      // dy2: nullable; a second gradient of y, added to dy (bf16 rounding of the sum)
    const void *y, *mbits, *x2;    // the ReLU mask: the forward's bits, else y (has_residual) or x; x2: sc's input
    void *dx, *dres, *ws;          // dres: the masked gradient (nullable), or with sc its input gradient (required)
    const BnLayer *bn, *sc;
    long long M;
    int C, relu, has_residual, reduced;   // reduced: dy's sums are in bn->dbeta / dgamma, the element-wise pass alone
};
cudaError_t launch_bn_bwd(const BnBwdPlan& b, cudaStream_t stream);
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
// rows of the statistics pass: passes of kBnRows rows, ppc passes per CTA (a multiple of kBnStatsUnroll), R CTAs
void bn_stats_plan(long long M, int C, long long* passes, long long* ppc, int* R);
// the same of the backward reduction pass (a multiple of kBnBwdReduceUnroll passes per CTA)
void bn_bwd_reduce_plan(long long M, int C, long long* passes, long long* ppc, int* R);
// the statistics pass alone (bn_stats_kernel): bn's save_mean / save_invstd and running statistics
cudaError_t launch_bn_stats(const void* x, long long M, int C, const BnLayer& bn, void* ws, cudaStream_t stream);
size_t conv1x1_workspace_bytes();
// the shapes each 1x1-convolution launcher takes (it returns cudaErrorNotSupported outside them)
bool conv1x1_stats_shape_ok(long long M, int Cin, int Cout);
bool conv1x1_apply_shape_ok(long long M, int Cin, int Cout);
bool conv1x1_dgrad_shape_ok(long long M, int Cin, int Cout);
cudaError_t launch_conv1x1_bn_stats(const void* x, const void* w, void* y, long long M, int Cin, int Cout,
                                    const BnLayer& bn, void* ws, cudaStream_t stream);
// y = relu(bn(x . w^T) + r) recomputing the convolution (moco_conv1x1_bn_add_relu_fwd); given as in BnFwdPlan
cudaError_t launch_conv1x1_bn_add_relu(const void* x, const void* w, const void* res, void* y, void* mask, long long M,
                                       int Cin, int Cout, const BnLayer& bn, const BnLayer* sc, int given, void* ws,
                                       cudaStream_t stream);
// dgrad of a 1x1 convolution, g = mask . bf16(bf16(dH . w) + dy2), and the backward sums of the BatchNorm that
// produced the convolution's input (moco_conv1x1_dgrad_bn_bwd)
cudaError_t launch_conv1x1_dgrad_bn_bwd(const void* dh, const void* w, void* g, long long M, int Cin, int Cout,
                                        const void* x, const void* mask, const void* dy2, const BnLayer& bn, void* ws,
                                        cudaStream_t stream);
// kNN classification against a feature bank (knn_sm90.cu, moco_knn)
constexpr int kKnnMaxNq = 1024;
struct KnnWorkspace {
    unsigned int* status;          // [0] the largest candidate count, [1] a label outside [0, n_classes)
    unsigned int* count;           // [Nq] candidates per query
    float* thresh;                 // [Nq] the sweep-2 threshold
    float* slice_max;              // [Nq][n_slices] the sweep-1 slice maxima
    unsigned long long* cand;      // [Nq][cap] candidate keys
    long long n_slices, cap;
    size_t fixed, bytes;           // fixed: everything but the candidate lists
};
struct KnnPlan {
    const int* labels;
    const int* targets;            // nullable
    int Nq;
    long long Nb;
    int C, k, n_classes;
    float inv_T;
    int* top5;
    float* scores5;                // nullable
    int* nbr_idx;                  // nullable
    float* nbr_sim;                // nullable
    int* correct;                  // nullable
};
KnnWorkspace knn_carve(void* base, int Nq, long long Nb, long long cap);
bool knn_shape_ok(int Nq, long long Nb, int C, int k);
cudaError_t launch_knn(const void* q, const void* bank, const KnnPlan& p, const KnnWorkspace& ws, cudaStream_t stream);
bool augment_shape_ok(int n_crops, int out_h, int out_w);
cudaError_t launch_augment(const void* pixels, size_t pixels_bytes, const moco_aug_crop* crops, int n_crops, int out_h,
                           int out_w, const float norm[6], void* dst, int dst_dtype, float* crop_means,
                           cudaStream_t stream);
cudaError_t launch_resize_windows(const void* pixels, size_t pixels_bytes, const moco_resize_window* windows, int n,
                                  int out_h, int out_w, const float norm[6], void* dst, int dst_dtype,
                                  cudaStream_t stream);
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
// the C the wgmma kernels take (a multiple of 64 up to 256)
bool nce_tc_shape_ok(int C);
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
