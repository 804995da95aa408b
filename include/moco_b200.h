/*
 * moco_b200 -- C ABI of the H100-native MoCo contrastive hot path.
 *
 * This is the drop-in boundary (SURVEY.md §8b).  The reference (bl0/moco) is pure
 * Python on PyTorch and has no FFI of its own; each entry point below replaces
 * the PyTorch library calls of one reference function (cited per function,
 * paths relative to the reference checkout).  A binding needs nothing but raw
 * device pointers, sizes and a cudaStream_t -- see INTEGRATION.md for the
 * ctypes stub a maintainer of the reference would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in `_host`;
 *   - compute calls are asynchronous on `stream` (a cudaStream_t passed as
 *     void*), re-entrant, allocate nothing and keep no global state besides the
 *     cached cuTensorMapEncodeTiled entry point and the launch counter
 *     (moco_launch_count); they are CUDA-graph capturable;
 *   - return value: 0 on success, a negative MOCO_ERR_* otherwise;
 *     moco_last_error() returns a thread-local human readable message;
 *   - row-major everywhere; `queue` is the [K, C] MoCo memory bank.
 */
#ifndef MOCO_B200_H
#define MOCO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MOCO_B200_ABI_VERSION 3 /* 3: + moco_bn_*, moco_maxpool3x3s2_*, moco_crop_s2d_bf16, moco_conv1x1_*,
                                    moco_augment_crops, moco_launch_count, moco_resize_center_crops,
                                    moco_augment_crops_blur (additive) */

enum {
    MOCO_OK = 0,
    MOCO_ERR_INVALID = -1,     /* bad argument (null pointer, size, alignment)          */
    MOCO_ERR_UNSUPPORTED = -2, /* valid but not implemented for this shape/dtype/device */
    MOCO_ERR_WORKSPACE = -3,   /* workspace too small                                    */
    MOCO_ERR_CUDA = -4,        /* a CUDA runtime/driver call failed                      */
    MOCO_ERR_CAPACITY = -5     /* moco_knn: a query has more candidates than the workspace holds */
};

enum { MOCO_F32 = 0, MOCO_BF16 = 1 };

/* moco_nce_fwd `flags` (0 = the tuned defaults).  Bit values 8, 16, 32, 64, 128 and 256 belonged to removed
 * kernel variants and stay reserved. */
enum {
    MOCO_NCE_AUTO = 0,         /* wgmma kernels when the shape allows it (C % 64 == 0, C <= 256)     */
    MOCO_NCE_FORCE_SIMT = 1,   /* generic CUDA-core kernel (any shape)                               */
    MOCO_NCE_CTA_PAIR = 2,     /* statistics kernel on 2-CTA clusters sharing each queue tile (TMA multicast) */
    MOCO_NCE_SINGLE_CTA = 4,   /* require the tensor-core path (error instead of the generic fallback) */
    MOCO_NCE_TWO_PASS = 512,   /* statistics pass, then dq pass normalised with the final lse (always exact) */
    MOCO_NCE_ONE_PASS = 1024   /* loss AND dq from one sweep over the queue (4NCK FLOP, NK exps instead of   */
                               /* 6NCK, 2NK) plus ONE tail kernel: every row stabilises with the constant    */
                               /* log2e * inv_T.  A row whose partial sum leaves the safe range (a logit     */
                               /* > ~100 binades above it, or all logits far below it: un-normalised         */
                               /* inputs) is detected by the tail kernel and recomputed exactly on CUDA      */
                               /* cores, so the result always equals the reference's.  AUTO picks it when dq */
                               /* is requested, logits are not, and inv_T <= MOCO_ONE_PASS_MAX_INV_T (with   */
                               /* L2-normalised q and queue rows of norm <= sqrt(3) -- the reference's       */
                               /* U(-s, s) initial queue, Contrast.py:16-17 -- the fallback never triggers); */
                               /* TWO_PASS otherwise.                                                         */
};
#define MOCO_ONE_PASS_MAX_INV_T 25.0f

int moco_abi_version(void);
const char* moco_last_error(void);

/* Number of SMs / compute capability of the current device (for tests & bench). */
int moco_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* Kernels this library has launched in this process, on all devices and threads: every kernel whose launch call
 * succeeded.  A launch recorded during stream capture counts once, when it is captured; replays of the graph do not
 * count. */
unsigned long long moco_launch_count(void);

/* ------------------------------------------------------------------------
 * InfoNCE head:  MemoryMoCo.forward logits (moco/NCE/Contrast.py:20-27) fused
 * with NCESoftmaxLoss (moco/NCE/NCECriterion.py:11-13), the `prob` metric
 * (train.py:264) and -- optionally, in the same pass over the queue -- the
 * gradient autograd would produce at train.py:273.
 *
 *   x[i,0]   = <q_i, k_i> * inv_T                       (positive, column 0)
 *   x[i,1+j] = <bf16(q_i), queue_j> * inv_T             (K negatives)
 *   lse[i]   = log sum_j exp(x[i,j]);  loss_rows[i] = lse[i] - x[i,0];
 *   prob_rows[i] = exp(x[i,0] - lse[i]);  loss_prob = {mean loss, mean prob}
 *   dq[i]    = d(mean loss)/dq_i
 *            = inv_T / N * ( (p_i0 - 1) * k_i + sum_j p_i,1+j * queue_j ),  p = softmax(x)
 *              (gradient w.r.t. q only: k and the queue are detached, Contrast.py:21,25)
 *
 * q, k: [N, C] of `qk_dtype` (MOCO_F32 or MOCO_BF16).  queue: [K, C] bf16, the
 * PRE-enqueue snapshot (Contrast.py:25) -- call moco_queue_enqueue afterwards on
 * the same stream.  Because dq is produced here, before the enqueue, no clone of
 * the queue is ever needed (the reference clones it every step, Contrast.py:24-25).
 * The contractions run on wgmma tensor cores with bf16 operands (q is rounded
 * to bf16 when given as f32) and fp32 accumulation; the positive logit is
 * computed in fp32 from the inputs as given.
 * `logits` ([N, K+1] fp32, row stride K+1) may be NULL: then no logit ever
 * reaches HBM.  `dq` ([N, C] fp32) may be NULL.  lse / loss_rows / prob_rows:
 * [N] fp32; loss_prob: [2] fp32.  All reductions are deterministic (fixed
 * order, no float atomics).  q and queue_bf16 must be 16-byte aligned
 * (MOCO_ERR_INVALID otherwise, before any device access).
 * Every logit is fp32(fp32(dot) * inv_T), with dot the fp32-accumulated product:
 * when every partial sum of a dot is exact in fp32 (e.g. operands with few
 * power-of-two entries) the logits are bit-identical on every path.
 * ---------------------------------------------------------------------- */
size_t moco_nce_workspace_bytes(int N, int C, int K);

int moco_nce_fwd(const void* q, const void* k, int qk_dtype,
                 const void* queue_bf16, int N, int C, int K, float inv_T,
                 float* logits_or_null, float* lse, float* loss_rows, float* prob_rows,
                 float* loss_prob, float* dq_or_null,
                 void* workspace, size_t workspace_bytes, int flags, void* stream);

/* ------------------------------------------------------------------------
 * One MoCo head step in TWO launches: moco_nce_fwd (one-sweep mode, no dense
 * logits) fused with moco_queue_enqueue, i.e. MemoryMoCo.forward
 * (moco/NCE/Contrast.py:20-36) + NCESoftmaxLoss (NCECriterion.py:11-13) + `prob`
 * (train.py:264) + the gradient of train.py:273:
 *
 *   kernel 1  the q.Queue^T sweep on wgmma (reads q as given, no cast kernel);
 *   kernel 2  merge -> lse / loss / prob, weighted sum of the partial gradients -> dq,
 *             then queue[(index + i) mod K] = k_all[i] for i in [0, n_all), and the
 *             ring position advanced on the device when `index_dev` is given.
 *
 * normalize != 0: q, k and k_all arrive UN-normalised (the encoder's fc output,
 * moco/models/resnet.py:125-126,177-178); the rows are L2-normalised inside the
 * kernels exactly like the reference's Normalize layer (resnet.py:24-33,
 * x / sqrt(sum x^2)) and dq is the gradient w.r.t. the RAW q (the backward of the
 * normalisation is applied in kernel 2).  Supported for C in {64, 128}.
 *
 * index / index_dev: the ring position BEFORE the call, by value, or -- when
 * index_dev != NULL -- read from that device int64 and advanced there
 * ((index + n_all) mod K, Contrast.py:34) by kernel 2, so a CUDA graph capturing
 * this call replays correctly step after step.  queue_f32 may be NULL.
 * q, queue_bf16, queue_f32 and k_all must be 16-byte aligned (MOCO_ERR_INVALID
 * otherwise, before any device access).
 * Shapes outside the one-sweep envelope fall back to the moco_nce_fwd kernels
 * followed by the enqueue kernel, which then reads and advances index_dev
 * itself; normalize must be 0 there (MOCO_ERR_UNSUPPORTED otherwise).
 * ---------------------------------------------------------------------- */
int moco_nce_step(const void* q, const void* k, int qk_dtype, int normalize,
                  void* queue_bf16, float* queue_f32_or_null, int N, int C, int K, float inv_T,
                  const void* k_all, int k_all_dtype, int n_all, int64_t index, int64_t* index_dev_or_null,
                  float* lse, float* loss_rows, float* prob_rows, float* loss_prob, float* dq,
                  void* workspace, size_t workspace_bytes, int flags, void* stream);

/* Profiling hook (bench.py's roofline): while set, moco_nce_fwd records the CUDA
 * events `ev_start` / `ev_stop` (cudaEvent_t) on its stream immediately before /
 * after launching kernel `kernel` (MOCO_PROF_STATS: the q.Queue^T statistics
 * kernel; MOCO_PROF_DQ: the dq kernel).  Pass NULLs to clear.  Not thread-safe. */
enum { MOCO_PROF_STATS = 1, MOCO_PROF_DQ = 2 };   /* one-pass mode: its single kernel reports as MOCO_PROF_DQ */
int moco_prof_set_events(int kernel, void* ev_start, void* ev_stop);
/* Device-clock window of the LAST sweep kernel that ran on `workspace` (first CTA entry -> last CTA exit, %globaltimer,
 * microseconds): what the kernel's CTAs took, without the grid-launch and completion latency a CUDA-event pair around
 * a single kernel also contains.  Synchronises `stream`.  n_ctas: upper bound on the grid (the SM count). */
int moco_prof_sweep_window(const void* workspace, int n_ctas, float* us_out, void* stream);
/* Backward of the dense-logits compatibility API (MemoryMoCo.forward returning
 * `out`, then an arbitrary upstream gradient):
 *   dq_i = inv_T * ( g_i0 * k_i + sum_j g_i,1+j * queue_j ),  g = grad_logits [N, K+1] fp32.
 * `queue_bf16` must be the PRE-enqueue snapshot the forward saw. */
int moco_nce_bwd_dense(const float* grad_logits, const void* k, int k_dtype,
                       const void* queue_bf16, int N, int C, int K, float inv_T,
                       float* dq, void* stream);

/* ------------------------------------------------------------------------
 * FIFO enqueue (moco/NCE/Contrast.py:29-34):
 *   for i in [0, n_all): queue[(index + i) mod K] = k_all[i]
 * `index` is the write pointer BEFORE the call; the caller advances it
 * ((index + n_all) mod K, Contrast.py:34).  Writes the bf16 working queue and,
 * when non-NULL, the fp32 master copy (the checkpointed `memory` buffer,
 * Contrast.py:18).  Requires n_all <= K (SURVEY S10).  queue_bf16, queue_f32 and
 * k_all must be 16-byte aligned (MOCO_ERR_INVALID otherwise); the same holds for
 * shard_bf16, shard_f32 and k_all of moco_queue_enqueue_shard.
 * ---------------------------------------------------------------------- */
int moco_queue_enqueue(void* queue_bf16, float* queue_f32_or_null,
                       const void* k_all, int k_dtype, int n_all, int C, int64_t K,
                       int64_t index, void* stream);

/* ------------------------------------------------------------------------
 * Sharded queue (BASELINE configs[3]; SURVEY §8e): rank r keeps rows
 * [r*K/W, (r+1)*K/W) of the K-row ring ("block" layout) instead of a replica.
 * Every rank evaluates ALL W*N queries against its shard; two small collectives
 * (done by the caller with NCCL) stitch the softmax together:
 *
 *   moco_nce_shard_stats : q_all, k_all [Nq, C] (Nq = W*N, rank-major), shard [Ks, C]
 *                          -> ms_out[Nq] float2 = per-row (max, sum 2^(x-max)) over the shard, log2 domain;
 *                          also leaves <q_i, k_i> and bf16(q_all) in the workspace
 *   ... all_gather ms_out -> ms_all [W, Nq] ...
 *   moco_nce_shard_merge : ms_all + the positive logit -> lse / loss_rows / prob_rows for all Nq rows
 *                          (same workspace as the stats call); loss_prob = means over all Nq rows
 *   moco_nce_shard_dq    : o_partial[Nq, C] = sum_{j in shard} exp(x_ij - lse_i) * shard_j
 *   ... reduce_scatter o_partial -> o_own [N, C] ...
 *   moco_nce_shard_dq_finish : dq_i = inv_T / N * (o_own_i + (prob_i - 1) * k_i)
 *
 * With MOCO_NCE_ONE_PASS in `flags` of BOTH moco_nce_shard_stats and
 * moco_nce_shard_dq, the statistics call makes the only sweep over the shard
 * (it also leaves the unnormalised P~.Queue partials in the workspace) and the
 * dq call just rescales and sums them with the merged lse -- the caller must not
 * use the workspace for anything else in between (moco_nce_shard_merge is fine).
 * Same numerical contract as MOCO_NCE_ONE_PASS of moco_nce_fwd: exact for any q.  A row one of whose slice
 * sums is above 2^100 or NaN, or whose shard sum is below 2^-80 (relative to the sweep's constant stabiliser
 * log2e * inv_T), is evaluated exactly on CUDA cores: the statistics call writes that row's exact
 * (log2 sum_{j in shard} 2^x_ij, 1) into ms_out and records the decision in the workspace, and the dq call
 * computes that row's o_partial exactly against the shard with the merged lse.  Same launches either way.
 *
 * moco_nce_shard_merge: world in [1, 160].  moco_nce_shard_dq_finish_peers: world in [1, 16], 0 <= rank < world,
 * every peer pointer non-NULL and 16-byte aligned, C a multiple of 4.
 *
 * The loss is permutation-invariant over negatives, so it equals the replicated
 * reference's; ring slot g of moco/NCE/Contrast.py:32 maps to (rank g / (K/W),
 * local row g % (K/W)) -- moco_queue_enqueue_shard writes only the slots this
 * rank owns, so indices stay checkable bit-exactly against the reference's.
 * ---------------------------------------------------------------------- */
int moco_nce_shard_stats(const void* q_all, const void* k_all, int qk_dtype, const void* shard_bf16,
                         int Nq, int C, int Ks, float inv_T, void* ms_out,
                         void* workspace, size_t workspace_bytes, int flags, void* stream);
int moco_nce_shard_merge(const void* ms_all, int world, int Nq, int C, float inv_T,
                         float* lse, float* loss_rows, float* prob_rows, float* loss_prob,
                         void* workspace, size_t workspace_bytes, void* stream);
int moco_nce_shard_dq(const void* q_all, int q_dtype, const void* shard_bf16, const float* lse_all,
                      int Nq, int C, int Ks, float inv_T, float* o_partial,
                      void* workspace, size_t workspace_bytes, int flags, void* stream);
int moco_nce_shard_dq_finish(const float* o_own, const void* k_own, int k_dtype,
                             const float* prob_rows_own, int N, int C, float inv_T, float* dq, void* stream);
/* The same last step with the reduce_scatter folded in: o_peers_host is a HOST array of `world` device pointers to
 * every rank's [world*N, C] fp32 o_partial (peer-mapped staging buffers, moco_p2p_*); this rank's rows
 * [rank*N, (rank+1)*N) of all of them are summed in rank order while dq is finished.  The caller orders the
 * peers' writes before this call with moco_signal_barrier. */
int moco_nce_shard_dq_finish_peers(const void* const* o_peers_host, int world, int rank, const void* k_own,
                                   int k_dtype, const float* prob_rows_own, int N, int C, float inv_T,
                                   float* dq, void* stream);
int moco_queue_enqueue_shard(void* shard_bf16, float* shard_f32_or_null, const void* k_all, int k_dtype,
                             int n_all, int C, int64_t K, int64_t index,
                             int64_t shard_row0, int64_t shard_rows, void* stream);

/* fp32 -> bf16 (round-to-nearest-even); used to (re)build the bf16 working queue
 * from the fp32 `memory` buffer (init / load_state_dict). */
int moco_f32_to_bf16(const float* src, void* dst_bf16, size_t n_elems, void* stream);

/* ------------------------------------------------------------------------
 * Momentum (EMA) update of the key encoder, ONE multi-tensor launch.  Replaces
 * moment_update (moco/util.py:124-127, called at train.py:277 and, with m = 0,
 * train.py:133):  for every parameter pair   p_ema = p_ema * m + (1 - m) * p,
 * evaluated per element as fma(one_minus_m, p, rn(p_ema * m)) -- bit-exact with
 * the reference's mul_ / add_(alpha) pair.
 *
 * segs_dev:         DEVICE array of n_segs records {float* p_ema; const float* p;
 *                   int64 n_elems;} (24 bytes each; an int64 [n_segs, 3] tensor).
 * chunk_prefix_dev: DEVICE int32 [n_segs + 1], exclusive prefix of
 *                   ceil(n_elems / moco_ema_chunk_elems()) per record;
 *                   n_chunks = chunk_prefix[n_segs].
 * The caller passes m and (1 - m) both already rounded to fp32 (the reference
 * computes 1 - m in double precision and rounds once).  fp32 tensors only. */
int moco_ema_chunk_elems(void);
int moco_ema_update(const void* segs_dev, const int32_t* chunk_prefix_dev, int n_segs, int n_chunks,
                    float m, float one_minus_m, void* stream);

/* ------------------------------------------------------------------------
 * Batch normalisation of the encoders' channels_last bf16 activations with the
 * block's ReLU and residual add folded in -- the consumer of ShuffleBN's output.
 * Replaces, at the reference's call sites moco/models/resnet.py:42-63 (BasicBlock),
 * :74-102 (Bottleneck), :114,156-157 (stem) and :139-143 (downsample), the sequence
 * nn.BatchNorm2d (training mode) [-> `out += residual`] [-> nn.ReLU]: per-channel
 * mean and biased variance over the M = N*H*W rows,
 *     y = relu?( (x - mean) * rsqrt(var + eps) * gamma + beta  [+ residual] ),
 * running_mean / running_var updated with `momentum` (unbiased variance), and
 * num_batches_tracked += 1, as torch.nn.BatchNorm2d does.  Arithmetic in fp32
 * from the bf16 inputs, one rounding to bf16 on output.
 *
 * x, residual, y, dy, dx, dresidual: bf16 [M, C] row-major (= NHWC storage), 16-byte
 * aligned, C a power of two in [64, 2048].  gamma, beta, running_*, save_*, dgamma,
 * dbeta: fp32 [C].  num_batches_tracked: int64 scalar on the device.  residual,
 * running_mean/var (both or neither) and num_batches_tracked may be NULL.
 * workspace: >= moco_bn_workspace_bytes() bytes, ZEROED ONCE by the caller before
 * its first use and then private to one stream (the kernels re-arm it).
 * Two launches per call (reduction + element-wise pass); deterministic.
 *
 * moco_bn_bwd: dy is the gradient w.r.t. y.  With g = dy masked by the ReLU
 * (mask recomputed from x when has_residual == 0 as y > 0 of the bf16 value the
 * forward stores, so a positive value that rounds to zero is off; read from y
 * otherwise -- y may be NULL unless relu && has_residual):  dbeta = sum g,  dgamma = sum g * x^,
 * dx = gamma * invstd * (g - dbeta / M - x^ * dgamma / M),  dresidual = g (written
 * only when dresidual != NULL).
 * ---------------------------------------------------------------------- */
size_t moco_bn_workspace_bytes(void);
int moco_bn_fwd_train(const void* x, const void* residual_or_null, void* y, long long M, int C,
                      const float* gamma, const float* beta, float* running_mean, float* running_var,
                      long long* num_batches_tracked, float momentum, float eps, int relu,
                      float* save_mean, float* save_invstd, void* workspace, size_t workspace_bytes, void* stream);
int moco_bn_bwd(const void* dy, const void* x, const void* y_or_null, long long M, int C,
                const float* gamma, const float* beta, const float* save_mean, const float* save_invstd,
                int relu, int has_residual, void* dx, void* dresidual_or_null, float* dgamma, float* dbeta,
                void* workspace, size_t workspace_bytes, void* stream);

/* The residual BatchNorm of a block, relu(bn(x) + r), with the ReLU mask kept as bits and, in a downsample block,
 * the shortcut's BatchNorm folded in.  Same arithmetic, roundings and reductions as moco_bn_fwd_train /
 * moco_bn_bwd: the results are bit-identical to those calls, with fewer bytes moved.
 *
 * moco_bn_layer: one BatchNorm's tensors.  gamma, beta, running_*, save_*, dgamma, dbeta: fp32 [C];
 * running_mean/var (both or neither) and num_batches_tracked may be NULL; momentum and eps as in
 * moco_bn_fwd_train.  The forward writes save_mean / save_invstd; the backward reads gamma and save_* and
 * writes dgamma / dbeta (beta, running_* and num_batches_tracked are not used there).
 *
 * moco_bn_add_relu_fwd_train: y = relu(bn(x) + r) with
 *     r = residual                                  when shortcut == NULL (identity shortcut),
 *     r = bf16(shortcut_bn(residual))               otherwise: residual is the shortcut convolution's raw output,
 *                                                   normalised with its own batch statistics (running statistics
 *                                                   updated as moco_bn_fwd_train does), rounded to bf16 as the
 *                                                   materialised shortcut output would be, and never written.
 *   mask (nullable; uint8 [M, C / 8]): bit k of byte (row, v) = (y[row, 8v + k] > 0), taken from the bf16 value of
 *   y as stored.  Write it when a backward follows.  Two launches (three with a shortcut BN).
 * moco_bn_add_relu_bwd: g = dy masked by `mask`.  dbeta = sum g, dgamma = sum g * x^, dx as moco_bn_bwd.  Without a
 *   shortcut BN, dresidual = g (nullable).  With one, the shortcut BN's backward runs in the same two passes on
 *   the same g: its dbeta = sum g, dgamma = sum g * residual^, and dresidual is its input gradient (required).
 *   Two launches.
 * x, residual, y, dy, dx, dresidual: bf16 [M, C] row-major, 16-byte aligned, C a power of two in [64, 2048];
 * workspace as for moco_bn_fwd_train (moco_bn_workspace_bytes() covers the three per-channel sums).
 * ---------------------------------------------------------------------- */
typedef struct moco_bn_layer {
    const float* gamma;
    const float* beta;
    float* running_mean;
    float* running_var;
    long long* num_batches_tracked;
    float momentum;
    float eps;
    float* save_mean;
    float* save_invstd;
    float* dgamma;
    float* dbeta;
} moco_bn_layer;

int moco_bn_add_relu_fwd_train(const void* x, const void* residual, void* y, void* mask_or_null, long long M, int C,
                               const moco_bn_layer* bn, const moco_bn_layer* shortcut_or_null,
                               void* workspace, size_t workspace_bytes, void* stream);
int moco_bn_add_relu_bwd(const void* dy, const void* x, const void* residual, const void* mask, long long M, int C,
                         const moco_bn_layer* bn, const moco_bn_layer* shortcut_or_null, void* dx,
                         void* dresidual_or_null, void* workspace, size_t workspace_bytes, void* stream);
/* moco_bn_add_relu_bwd2: moco_bn_add_relu_bwd with y's gradient arriving in two parts, dy and dy2 (bf16 [M, C]): the
 * input of the next block feeds both its first convolution and its residual branch.  Both passes read both and use
 * bf16(dy + dy2) (fp32 add, one rounding -- what a separate bf16 add would store), which is never written; the
 * results are bit-identical to that add followed by moco_bn_add_relu_bwd.  Two launches. */
int moco_bn_add_relu_bwd2(const void* dy, const void* dy2, const void* x, const void* residual, const void* mask,
                          long long M, int C, const moco_bn_layer* bn, const moco_bn_layer* shortcut_or_null, void* dx,
                          void* dresidual_or_null, void* workspace, size_t workspace_bytes, void* stream);

/* The training forward of moco_bn_fwd_train / moco_bn_add_relu_fwd_train for BatchNorms whose batch statistics are
 * already computed (moco_conv1x1_bn_stats): `stats_given` bit MOCO_BN_STATS_GIVEN says bn's save_mean / save_invstd
 * (and its running statistics) are final, MOCO_BN_SC_STATS_GIVEN the same of the shortcut BN.  A layer whose bit is
 * clear gets its statistics pass here, as in those calls; then one element-wise pass writes
 *     y = relu?(bn(x) [+ r]),   r = residual, or bf16(shortcut_bn(residual)) with a shortcut BN (residual required),
 * and the mask bits (nullable) as moco_bn_add_relu_fwd_train does.  Same apply kernel, so with the same statistics
 * the outputs are bit-identical to those calls.  workspace may be NULL when no statistics pass runs.  One launch plus
 * one per statistics pass. */
enum { MOCO_BN_STATS_GIVEN = 1, MOCO_BN_SC_STATS_GIVEN = 2 };
int moco_bn_fwd_train_given(const void* x, const void* residual_or_null, void* y, void* mask_or_null, long long M,
                            int C, int relu, const moco_bn_layer* bn, const moco_bn_layer* shortcut_or_null,
                            int stats_given, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * 1x1 / stride 1 convolution forward with the following training BatchNorm's batch statistics: in NHWC the
 * convolution is the GEMM  y[M, Cout] = x[M, Cin] . w[Cout, Cin]^T  (bf16 operands, fp32 accumulation, y rounded to
 * bf16 once), and the statistics are those of y as rounded, finished as moco_bn_fwd_train's statistics pass does
 * (mean and biased variance over the M rows, save_mean / save_invstd, running_mean / running_var with the unbiased
 * variance, num_batches_tracked += 1).  Only bn's running_*, num_batches_tracked, momentum, eps and save_* are used.
 * Follow it with moco_bn_fwd_train_given.  One launch on Hopper tensor cores (wgmma, TMA); deterministic.
 *
 * x: bf16 [M, Cin] (NHWC storage), w: bf16 [Cout, Cin] (the [Cout, Cin, 1, 1] weight), y: bf16 [M, Cout]; all
 * 16-byte aligned.  Cin a multiple of 64 in [64, 65536], Cout a multiple of 64 in [64, 4096], M >= 1.
 * workspace: >= moco_conv1x1_workspace_bytes() bytes, ZEROED ONCE before its first use, then private to one stream.
 * ---------------------------------------------------------------------- */
size_t moco_conv1x1_workspace_bytes(void);
int moco_conv1x1_bn_stats(const void* x, const void* w, void* y, long long M, int Cin, int Cout,
                          const moco_bn_layer* bn, void* workspace, size_t workspace_bytes, void* stream);

/* A block's residual BatchNorm on that convolution's output, y = relu(bn(x . w^T) + r), computed from the convolution's
 * INPUT x: the GEMM runs again with the BatchNorm, the add and the ReLU in its epilogue, so the convolution's output h
 * is neither written nor read here.  r as in moco_bn_fwd_train_given (residual, or bf16(shortcut_bn(residual)) with a
 * shortcut BN).  With the same statistics, y and the mask bits are bit-identical to moco_conv1x1_bn_stats followed by
 * moco_bn_fwd_train_given (relu = 1): the recomputed tile is, by construction, the h that call stores.
 *   stats_given bit MOCO_BN_STATS_GIVEN set: bn's statistics are final (moco_conv1x1_bn_stats ran; a backward that
 *     needs h has it from there).  Clear: moco_conv1x1_bn_stats's pass runs first WITHOUT storing h -- for a forward
 *     with no backward, where h is never needed.
 *   MOCO_BN_SC_STATS_GIVEN clear with a shortcut BN: its statistics pass over residual runs first.
 * x: bf16 [M, Cin], w: bf16 [Cout, Cin], residual, y: bf16 [M, Cout], mask (nullable): uint8 [M, Cout / 8]; pointers
 * 16-byte aligned.  Cin a multiple of 64 in [64, 65536], Cout a power of two in [64, 2048], 1 <= M < 2^31 - 128.
 * workspace: zeroed once, private to one stream, at least the larger of moco_conv1x1_workspace_bytes() and
 * moco_bn_workspace_bytes() when a statistics pass runs (NULL otherwise allowed).  One launch plus one per statistics
 * pass. */
int moco_conv1x1_bn_add_relu_fwd(const void* x, const void* w, const void* residual, void* y, void* mask_or_null,
                                 long long M, int Cin, int Cout, const moco_bn_layer* bn,
                                 const moco_bn_layer* shortcut_or_null, int stats_given, void* workspace,
                                 size_t workspace_bytes, void* stream);

/* The backward of that convolution when its input is the output of a block's residual BatchNorm (moco_bn_add_relu_*,
 * identity shortcut) whose gradient also has a second part dy2 (the next block's residual branch): the input gradient
 * of the convolution taken with that BatchNorm's backward reduction.  One launch; deterministic.
 *   dX = dh . w  (dh: bf16 [M, Cout], the gradient of the convolution's output; fp32 accumulation, rounded to bf16),
 *   g  = mask . bf16(dX + dy2)   -- the masked gradient moco_bn_add_relu_bwd2 forms from dy = dX and dy2,
 *   bn->dbeta = sum g,  bn->dgamma = sum g * x^   -- bit-identical to moco_bn_add_relu_bwd2's given the same dX.
 * g (bf16 [M, Cin]) is written: it is also the residual gradient of an identity block.  Follow it with
 * moco_bn_bwd_apply_given.  x: that BatchNorm's input, bf16 [M, Cin]; mask: its forward's mask bytes (uint8
 * [M, Cin / 8]); only bn's save_mean, save_invstd, dgamma and dbeta are used.  Cin a power of two in [128, 2048],
 * Cout a multiple of 64 in [64, 4096], 1 <= M < 2^31 - 128; pointers 16-byte aligned.  mask and dy2 are required
 * and x2 / shortcut must be NULL: the other producers (a downsample block's bn3, a BatchNorm without residual) are
 * MOCO_ERR_UNSUPPORTED.  workspace as for moco_conv1x1_bn_stats. */
int moco_conv1x1_dgrad_bn_bwd(const void* dh, const void* w, void* g, long long M, int Cin, int Cout, const void* x,
                              const void* mask, const void* dy2, const void* x2_or_null,
                              const moco_bn_layer* bn, const moco_bn_layer* shortcut_or_null, void* workspace,
                              size_t workspace_bytes, void* stream);
/* The element-wise pass of the BatchNorm backward alone, on an already-masked gradient g whose sums are in bn->dbeta /
 * bn->dgamma: dx as moco_bn_bwd.  Bit-identical to the second pass of moco_bn_add_relu_bwd(2) given the same g and
 * sums.  One launch, no workspace.  g, x, dx: bf16 [M, C], 16-byte aligned, C a power of two in [64, 2048].  A shortcut
 * BN (x2, dx2, shortcut) is validated but not implemented: MOCO_ERR_UNSUPPORTED. */
int moco_bn_bwd_apply_given(const void* g, const void* x, const void* x2_or_null, long long M, int C,
                            const moco_bn_layer* bn, const moco_bn_layer* shortcut_or_null, void* dx,
                            void* dx2_or_null, void* stream);

/* ------------------------------------------------------------------------
 * Weighted k-nearest-neighbour classification against a feature bank (the kNN monitor of instance discrimination,
 * lemniscate.pytorch's kNN with its weights exp(s / T)), without storing the [Nq, Nb] similarity matrix.
 *
 * q: bf16 [Nq, C], 1 <= Nq <= 1024; bank: bf16 [Nb, C], k <= Nb < 2^31 (it may pass 2^32 bytes); C a multiple of 64 in
 * [64, 2048]; both 16-byte aligned.  labels: int32 [Nb], each in [0, n_classes); n_classes in [1, 65536]; k in
 * [1, 1024]; inv_T = 1 / T > 0.
 *   s(i, j) = the fp32 dot product of q_i and bank_j (wgmma, fp32 accumulation in increasing C; exact whenever the
 *   products' partial sums are exact in fp32).
 *   N(i) = the first k bank rows under the total order (s descending, j ascending): the result depends on nothing else,
 *   not on the grid, the workspace or the timing.
 *   score(i, c) = sum over j in N(i) with labels[j] = c of exp((s(i, j) - s_max(i)) * inv_T), s_max(i) = the largest
 *   s(i, j); fp32, each class's terms added in N(i)'s order.  Subtracting s_max changes no prediction.
 *   The predictions are the classes in the order (score descending, class ascending): top5 int32 [Nq, 5] (-1 past
 *   n_classes), scores5 (nullable) fp32 [Nq, 5] their scores.
 * nbr_idx / nbr_sim (nullable): int32 / fp32 [Nq, k], N(i) in order and its similarities.  targets (nullable) int32
 * [Nq] with correct int32 [2]: correct = {#(top5[i][0] == target_i), #(target_i in top5[i])}, over this call.
 * Outputs may not overlap one another, the inputs or the workspace.  Non-finite features are outside this contract.
 *
 * workspace: 256-byte aligned, moco_knn_workspace_bytes(Nq, Nb, capacity) bytes for room for `capacity` candidates
 * per query (the call uses all it is given, up to Nb); at least capacity = k, else MOCO_ERR_WORKSPACE.  A query's
 * candidates are the rows with s at least a lower bound on its k-th largest similarity: a few times k for spread
 * similarities, up to Nb when many rows tie.  When a query has more than the workspace holds, the call returns
 * MOCO_ERR_CAPACITY; the outputs are then undefined, nothing is truncated, and a call with
 * moco_knn_workspace_bytes(Nq, Nb, *need_capacity) bytes gives the answer.
 * need_capacity (HOST): the largest candidate count of any query, also on success.  A label outside [0, n_classes)
 * among the neighbours is reported after the fact as MOCO_ERR_INVALID.
 *
 * Four launches (the two sweeps over the bank on Hopper tensor cores, a threshold kernel, a select-and-vote kernel),
 * then the call synchronises `stream` to read the candidate counts: it is not graph-capturable.  Needs sm_90.
 * ---------------------------------------------------------------------- */
size_t moco_knn_workspace_bytes(int Nq, long long Nb, long long capacity);
int moco_knn(const void* q, const void* bank, const int32_t* labels, int Nq, long long Nb, int C, int k, float inv_T,
             int n_classes, const int32_t* targets_or_null, int32_t* top5, float* scores5_or_null,
             int32_t* nbr_idx_or_null, float* nbr_sim_or_null, int32_t* correct_or_null, void* workspace,
             size_t workspace_bytes, long long* need_capacity, void* stream);

/* The stem's BatchNorm + ReLU followed by its 3x3 / stride 2 / pad 1 max pooling, without writing the BatchNorm's
 * output: bit-identical to moco_bn_fwd_train (relu = 1, no residual) + moco_maxpool3x3s2_fwd.  The statistics pass,
 * then one pass that applies BatchNorm + ReLU to every tap (rounded to bf16 as the BatchNorm's own pass stores it)
 * and takes the max by torch's rule.  Two launches.
 * x: bf16 [N, H, W, C] (NHWC storage), the BatchNorm's input, C a power of two in [64, 2048]; y, taps: the pooled
 * output and the winning tap bytes as moco_maxpool3x3s2_fwd defines them; workspace as for moco_bn_fwd_train.
 * The backward is moco_maxpool3x3s2_bwd followed by moco_bn_bwd (relu = 1, has_residual = 0), which recomputes the
 * ReLU mask from x. */
int moco_bn_relu_maxpool_fwd_train(const void* x, void* y, void* taps_u8, int N, int H, int W, int C,
                                   const moco_bn_layer* bn, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Frozen (eval-mode) BatchNorm for the linear probe's encoder forward (the reference's eval.py runs the pretrained
 * ResNet in eval mode): the same groups as above with the running statistics folded into two per-channel fp32
 * vectors by the caller,
 *     scale = gamma / sqrt(running_var + eps),   shift = beta - running_mean * scale,
 * so there is no statistics pass and no backward.  One launch each, no workspace.
 *
 * Numerical contract (fp32, every operation rounded to nearest, NO fused multiply-add; it therefore differs from the
 * training apply pass, which uses fmaf, and is reproduced exactly by separate fp32 torch ops):
 *     z = (x * scale) + shift
 *     z = z + r                                          when there is a residual
 *     z = z > 0 ? z : 0                                  when relu
 *     y = bf16_rn(z)
 * with r = residual, or with a shortcut BN r = bf16_rn((residual * sc_scale) + sc_shift): residual is then the
 * shortcut convolution's raw output, rounded as its materialised BatchNorm output would be, and never written.
 * The average pool: feat[n, c] = (sum over p = 0 .. HW-1 of f32(y[n, p, c]), added in increasing p) / HW, with
 * y the bf16-rounded value and one IEEE division.
 *
 * x, residual, y: bf16 [M, C] row-major (NHWC storage), 16-byte aligned, C a power of two in [64, 2048];
 * scale, shift, sc_scale, sc_shift: fp32 [C]; sc_scale / sc_shift both or neither, and only with a residual.
 *
 * moco_bn_eval_act: y = relu?(bn(x) [+ r]), bf16 [M, C].
 * moco_bn_relu_maxpool_eval: the stem, relu(bn(x)) (relu always on) applied to each tap of the 3x3 / stride 2 / pad 1
 *   max pool of moco_maxpool3x3s2_fwd, x [N, H, W, C] -> y [N, OH, OW, C]; no tap bytes are written.
 * moco_bn_eval_act_avgpool: the last block's group followed by the global average pool, x [N, HW, C] ->
 *   feat fp32 [N, C] (16-byte aligned); the [N, HW, C] map is never written.
 * ---------------------------------------------------------------------- */
int moco_bn_eval_act(const void* x, const void* residual_or_null, void* y, long long M, int C, const float* scale,
                     const float* shift, int relu, const float* sc_scale_or_null, const float* sc_shift_or_null,
                     void* stream);
int moco_bn_relu_maxpool_eval(const void* x, void* y, int N, int H, int W, int C, const float* scale,
                              const float* shift, void* stream);
int moco_bn_eval_act_avgpool(const void* x, const void* residual_or_null, float* feat_f32, int N, int HW, int C,
                             const float* scale, const float* shift, int relu, const float* sc_scale_or_null,
                             const float* sc_shift_or_null, void* stream);

/* The same input pass (crop of the [N, C_total >= 3, H, W] batch, optional row permutation, cast to bf16) written in
 * the layout of a space-to-depth stem: dst = bf16 [N, H/2 + 3, W/2 + 3, 16] with
 *     dst[n, R, Q, (b * 2 + d) * 3 + c] = src[rows[n], c, 2 (R - 2) + b, 2 (Q - 2) + d]   (0 outside; channels 12..15 = 0)
 * over which the reference's first convolution (moco/models/resnet.py:112: 7x7, stride 2, padding 3, 3 -> 64) is a
 * 4x4 / stride 1 / padding 0 convolution with the re-indexed weights w'[o, (b*2+d)*3+c, a, e] = w[o, c, 2a+b-1, 2e+d-1]
 * (moco_b200/encoders.py:StemConv).  H, W even; src fp32 (8-byte aligned rows) or bf16.  src_rows may be NULL. */
int moco_crop_s2d_bf16(const void* src, int src_dtype, long long src_image_stride, const int64_t* src_rows_or_null,
                       void* dst_bf16, int N, int H, int W, void* stream);

/* ------------------------------------------------------------------------
 * The stem's max pooling on channels_last bf16 activations.  Replaces
 * `nn.MaxPool2d(kernel_size=3, stride=2, padding=1)` (moco/models/resnet.py:119,158)
 * and its backward.  x: bf16 [N, H, W, C] (NHWC storage), C % 8 == 0;
 * y: bf16 [N, OH, OW, C] with OH = (H - 1) / 2 + 1, OW = (W - 1) / 2 + 1;
 * taps: uint8 [N, OH, OW, C], the winning tap kh * 3 + kw of every output element
 * (first maximum in kh-then-kw order, NaN wins -- torch's rule), written by the
 * forward and consumed by the backward, which adds dy into the winning input
 * element of every window (gather over the <= 4 windows of a pixel: no atomics,
 * deterministic, fp32 sums in increasing (oh, ow) order).  N <= 65535.  One launch each.
 * moco_maxpool3x3s2_bwd2: the backward with the pooled output's gradient in two parts, dy and dy2 (the stem's output
 * feeds the first block's convolution and its residual branch): each window's gradient is bf16(dy + dy2), the value a
 * separate bf16 add would store, never written; bit-identical to that add followed by moco_maxpool3x3s2_bwd.
 * ---------------------------------------------------------------------- */
int moco_maxpool3x3s2_fwd(const void* x, void* y, void* taps_u8, int N, int H, int W, int C, void* stream);
int moco_maxpool3x3s2_bwd(const void* dy, const void* taps_u8, void* dx, int N, int H, int W, int C, void* stream);
int moco_maxpool3x3s2_bwd2(const void* dy, const void* dy2, const void* taps_u8, void* dx, int N, int H, int W, int C,
                           void* stream);

/* ------------------------------------------------------------------------
 * Input path (SURVEY.md 8 f3): one crop of the [N, C_total, H, W] batch ->
 * bf16 [N, H, W, C] (channels_last storage) in ONE pass.  Replaces the crop
 * split of train.py:250-254 (`torch.split(inputs, [3, 3], dim=1)` + the
 * discarded `.contiguous()` calls) and the cast + layout passes mixed
 * precision / cuDNN put in front of the first convolution.
 *
 * src: MOCO_F32 or MOCO_BF16, NCHW, pointing at the crop's first channel of
 * image 0; `src_image_stride` = ELEMENTS between consecutive images (C_total *
 * H*W, so a crop is read in place from the 6-channel batch).  dst: dense
 * [N, H*W, C] bf16.  C <= 4, H*W a multiple of 8, src 16-byte aligned.
 * Values are rounded to nearest-even bf16 -- bit-identical to torch's
 * `.to(torch.bfloat16)`. */
int moco_crop_to_nhwc_bf16(const void* src, int src_dtype, long long src_image_stride, void* dst_bf16,
                           int N, int C, int HW, void* stream);

/* The same with a row permutation: dst image i = crop of src image src_rows[i] (device int64 [N]; NULL = identity).
 * On ONE GPU this is the whole ShuffleBN forward permute (moco/util.py:69-79) fused with the input path: the
 * permutation is the address computation of the one pass over the images. */
int moco_crop_gather_nhwc_bf16(const void* src, int src_dtype, long long src_image_stride, const int64_t* src_rows,
                               void* dst_bf16, int N, int C, int HW, void* stream);

/* ------------------------------------------------------------------------
 * Data augmentation of the two pre-training crops (train.py:106-114 applied twice per image, moco/dataset.py:25-33)
 * from decoded uint8 images: the loader's workers only decode and draw the random parameters, and the device receives
 * the source pixels instead of fp32 [N, 6, 224, 224] crops.
 *
 * Crop i is torchvision's TENSOR implementation (torchvision.transforms.functional) of the reference's transform,
 * applied to x = src_uint8 / 255 in fp32, with the parameters of record crops[i]:
 *   1. resized_crop(x, top, left, height, width, [out_h, out_w], antialias=True): ATen's upsample_bilinear2d_aa,
 *      triangle filter of support max(scale, 1), taps clipped at the crop's border, weights renormalised;
 *   2. rgb_to_grayscale(x, 3) (0.2989 r + 0.587 g + 0.114 b) when flags has MOCO_AUG_GRAY;
 *   3. when flags has MOCO_AUG_JITTER, for k = 0..3 op (order >> 2k) & 3 (ColorJitter's fn_idx):
 *      0 adjust_brightness, 1 adjust_contrast, 2 adjust_saturation, 3 adjust_hue with the record's factors;
 *      _blend(a, b, r) = clamp(r a + (1 - r) b, 0, 1); the contrast mean is the mean grayscale of the whole crop as it
 *      stands before the contrast op; hue via _rgb2hsv / _hsv2rgb with the shifted hue taken % 1.0;
 *   4. hflip when flags has MOCO_AUG_FLIP;
 *   5. (x - mean[c]) / std[c], a subtraction then a division (norm_host = {mean[3], std[3]}, a HOST array).
 * Every step is fp32 in torchvision's operation order, with three deviations in the resample: the vertical pass runs
 * first (ATen's CPU kernel runs the horizontal one first), it sums the raw uint8 values and divides by 255 after
 * the pass, and each weight is scaled by the correctly rounded reciprocal of the weights' sum instead of divided by
 * it.  So results agree with torchvision to fp32 rounding, not bit for bit; oracle/augment_oracle.py restates the
 * exact order, which the kernels match bit for bit, the contrast mean's reduction order included.  The
 * reference itself runs PIL on uint8, which rounds after every step: this is the documented deviation from it.
 *
 * pixels: packed uint8 HWC RGB images, image of crop i at byte crops[i].src_offset (src_h * src_w * 3 bytes).
 * crops: DEVICE array of n_crops records.  dst: crop i at dst + i * 3 * out_h * out_w elements, three NCHW planes,
 * MOCO_F32 or MOCO_BF16 (the round-to-nearest-even of the fp32 value): a [2N, 3, H, W] tensor of crops
 * (2n, 2n + 1) of image n is the reference's [N, 6, H, W] batch.  crop_means: DEVICE float [n_crops] scratch (the
 * contrast means).  out_h, out_w in [1, 1024]; n_crops in [0, 65535]; a crop at most 1000 * out_w pixels wide.
 * The records are validated on the host by the caller (moco_b200/augment.py); here every source index is clamped
 * into its own image and into [0, pixels_bytes), so a malformed record gives unspecified values but never reads
 * outside the buffer.  Two launches (the contrast means, then the crops); deterministic.
 * ---------------------------------------------------------------------- */
enum { MOCO_AUG_GRAY = 1, MOCO_AUG_FLIP = 2, MOCO_AUG_JITTER = 4 };
typedef struct moco_aug_crop {
    int64_t src_offset;                   /* byte offset of the source image in `pixels`                 */
    int32_t src_h, src_w;                 /* source image size                                           */
    int32_t top, left, height, width;     /* crop box (RandomResizedCrop.get_params: i, j, h, w)         */
    int32_t flags;                        /* MOCO_AUG_*                                                  */
    int32_t order;                        /* ColorJitter's fn_idx, op k in bits 2k..2k+1                 */
    float brightness, contrast, saturation, hue;
} moco_aug_crop;                          /* 56 bytes                                                    */

int moco_augment_crops(const void* pixels, size_t pixels_bytes, const moco_aug_crop* crops, int n_crops, int out_h,
                       int out_w, const float* norm_host, void* dst, int dst_dtype, float* crop_means, void* stream);

/* ------------------------------------------------------------------------
 * The MoCo v2 augmentation ("aug-plus"): RandomResizedCrop -> RandomApply(ColorJitter, 0.8) -> RandomGrayscale ->
 * RandomApply(GaussianBlur(ksize, sigma), 0.5) -> RandomHorizontalFlip -> Normalize, in the conventions of
 * moco_augment_crops above.  Each record is a moco_aug_crop followed by two switches and the blur's weights:
 *   1. the resample, as moco_augment_crops;
 *   2. rgb_to_grayscale when flags has MOCO_AUG_GRAY and gray_after_jitter == 0;
 *   3. the jitter, as moco_augment_crops (flags MOCO_AUG_JITTER, order, factors);
 *   4. rgb_to_grayscale when flags has MOCO_AUG_GRAY and gray_after_jitter != 0 (the v2 order);
 *   5. when blur != 0, torchvision's tensor gaussian_blur with the 1-D kernel k[j] = weights[|j - h|], j = 0 .. 2h,
 *      h = ksize / 2: reflect padding of h on the crop as it stands after step 4 (row -i is row i, row out_h - 1 + i
 *      is row out_h - 1 - i; columns likewise), then
 *          t(y, x)   = sum for j = 0 .. 2h of k[j] * s(reflect(y - h + j), x)     (vertical pass first)
 *          out(y, x) = sum for j = 0 .. 2h of k[j] * t(y, reflect(x - h + j))     (then the horizontal pass)
 *      each sum started from 0 and taken in tap order j, every product and addition one fp32 operation rounded to
 *      nearest.  The blur runs in unflipped coordinates, before the flip;
 *   6. hflip when flags has MOCO_AUG_FLIP, then Normalize.
 * The contrast mean is that of moco_augment_crops: the mean grayscale before the contrast op, before any blur.
 * torchvision's conv2d sums the rounded 2-D products ky[a] * kx[b] in its own order, so the blurred crops, too, agree
 * with torchvision to fp32 rounding; tests/augment_blur_oracle.py restates this order and the kernels match it bit
 * for bit.  With blur = 0 and gray_after_jitter = 0 a record computes exactly what moco_augment_crops computes.
 *
 * weights: the half kernel kernel1d[h], kernel1d[h + 1], ..., kernel1d[2h], zero past index h.  The caller computes
 * them on the host with torchvision's _get_gaussian_kernel1d arithmetic (linspace, exp(-0.5 (x / sigma)^2), / sum, in
 * fp32), which is symmetric bit for bit for an odd ksize; the device evaluates no transcendental function.
 * ksize: odd, in [3, 31], ksize / 2 < min(out_h, out_w) (reflect padding needs it); one per call.
 * out_h, out_w in [1, 512]; n_crops in [0, 65535]; a crop at most 1000 * out_w pixels wide.  Anything outside this
 * envelope is refused before any launch.  crops: DEVICE array, 8-byte aligned.  A malformed record gives unspecified
 * values but never reads outside the pixel buffer or shared memory: source indices are clamped as in
 * moco_augment_crops, the two switches are tested against 0 and the weights are only multiplied.
 *
 * Three launches, each over all n_crops records: the contrast means; the apply pass of the unblurred crops (8 output
 * rows per CTA, as moco_augment_crops; a blurred crop's CTAs exit at once); the apply pass of the blurred crops, each
 * CTA a band of up to 32 output rows at full width that evaluates steps 1-4 for its rows and the h rows either side
 * into shared memory as fp32 RGB and blurs out of it (an unblurred crop's CTAs exit at once).  Deterministic.
 * ---------------------------------------------------------------------- */
typedef struct moco_aug_crop_blur {
    moco_aug_crop crop;                   /* the moco_aug_crop record, unchanged in meaning              */
    int32_t gray_after_jitter;            /* 0: grayscale before the jitter (v1), else after it (v2)     */
    int32_t blur;                         /* 0: no blur                                                  */
    float weights[16];                    /* the half kernel, kernel1d[h + i]; zero past i = h           */
} moco_aug_crop_blur;                     /* 128 bytes                                                   */

int moco_augment_crops_blur(const void* pixels, size_t pixels_bytes, const moco_aug_crop_blur* crops, int n_crops,
                            int out_h, int out_w, int ksize, const float* norm_host, void* dst, int dst_dtype,
                            float* crop_means, void* stream);

/* ------------------------------------------------------------------------
 * The validation transform of the linear evaluation (eval.py:111-116: Resize(256) -> CenterCrop(224) -> ToTensor ->
 * Normalize) from decoded uint8 images, in the conventions of moco_augment_crops above.
 *
 * Output image i is torchvision's TENSOR implementation applied to x = src_uint8 / 255 in fp32, with record
 * windows[i]:
 *   1. resize(x, [resized_h, resized_w], antialias=True): ATen's upsample_bilinear2d_aa of the WHOLE source image;
 *   2. rows [top, top + out_h) and columns [left, left + out_w) of the resized image (center_crop's window).  Only the
 *      window is computed: the resized image is never materialised;
 *   3. (x - mean[c]) / std[c] (norm_host = {mean[3], std[3]}, a HOST array).
 * The host fills the record with torchvision's arithmetic (moco_b200.augment.resize_window_params): Resize(int) keeps
 * the short side at `resize` and sets the long side to int(resize * long / short); CenterCrop's offset is
 * int(round((resized - out) / 2.0)), Python's round half to even.  Same fp32 operation order and the same deviation
 * from PIL as moco_augment_crops; results agree with torchvision to fp32 rounding.
 *
 * pixels: packed uint8 HWC RGB images, image i at byte windows[i].src_offset.  windows: DEVICE array of n records.
 * dst: image i at dst + i * 3 * out_h * out_w elements, MOCO_F32 or MOCO_BF16 (round-to-nearest-even of the fp32
 * value): an [n, 3, out_h, out_w] tensor.  out_h, out_w in [1, 1024]; n in [0, 65535]; a source at most
 * 1000 * resized_w pixels wide.  The records are validated on the host by the caller; here the window is clamped into
 * the resized image and every source index into its own image and into [0, pixels_bytes), so a malformed record gives
 * unspecified values but never reads outside the buffer.  One launch; deterministic.
 * ---------------------------------------------------------------------- */
typedef struct moco_resize_window {
    int64_t src_offset;                   /* byte offset of the source image in `pixels`                 */
    int32_t src_h, src_w;                 /* source image size                                           */
    int32_t resized_h, resized_w;         /* size of the resized image the window is taken from          */
    int32_t top, left;                    /* window origin in the resized image                          */
} moco_resize_window;                     /* 32 bytes                                                    */

int moco_resize_center_crops(const void* pixels, size_t pixels_bytes, const moco_resize_window* windows, int n,
                             int out_h, int out_w, const float* norm_host, void* dst, int dst_dtype, void* stream);

/* ------------------------------------------------------------------------
 * ShuffleBN row gather over NVLink peer memory.  Replaces dist_collect +
 * fancy-index (moco/util.py:47-58,74-79,88-91): instead of all_gather-ing every
 * rank's batch and indexing, each rank pulls exactly the rows it needs.
 *
 *   for i in [0, n_rows): g = src_rows[i];
 *       dst[i] = peer_base_host[g / rows_per_rank] + (g % rows_per_rank) * row_bytes
 *
 * peer_base_host: HOST array of `world` device pointers (peer-mapped buffers from
 * moco_p2p_* below; world = 1 -> the local buffer).  src_rows: DEVICE int64
 * [n_rows] global row ids (the slice of forward_inds / backward_inds this rank
 * needs, util.py:77,91).  row_bytes must be a multiple of 16 and buffers 16-byte
 * aligned.  Synchronisation with the peers (data ready / buffer reusable) is the
 * caller's: moco_signal_barrier.
 * flags: MOCO_GATHER_AUTO = bulk-async (TMA) copies for rows of 16 KiB .. 400 KiB,
 * the 16-byte load/store kernel above that (measured faster for fp32 image rows), one
 * warp per row below; MOCO_GATHER_LDG = always the load/store kernel for large rows.
 * ---------------------------------------------------------------------- */
enum { MOCO_GATHER_AUTO = 0, MOCO_GATHER_LDG = 1 };
int moco_shuffle_gather(const void* const* peer_base_host, int world, int rows_per_rank,
                        const int64_t* src_rows, int n_rows, size_t row_bytes,
                        void* dst, int flags, void* stream);

/* The same gather with the cross-GPU synchronisation folded into the SAME kernel (ShuffleBN forward = publish + this
 * one launch): block 0 publishes "rank `rank` has finished writing its staging buffer" (event number `epoch`) into
 * every peer's signal pad, and every block waits until all `world` peers have published that event before its first
 * pull.  Pads and epoch numbering are those of moco_signal_barrier (one event = one epoch, whichever call carries it).
 * The wait is bounded in time (MOCO_BARRIER_TIMEOUT_MS, default 120000): on expiry the kernel records the reason in a
 * pinned status block (moco_p2p_last_timeout) and traps. */
int moco_shuffle_gather_sync(const void* const* peer_base_host, void* const* signal_pads_host, int world, int rank,
                             uint32_t epoch, int rows_per_rank, const int64_t* src_rows, int n_rows,
                             size_t row_bytes, void* dst, int flags, void* stream);

/* out[0] = 1 if a peer wait of this process timed out (0 otherwise), out[1] = the peer rank waited for,
 * out[2] = the event number, out[3] = milliseconds waited.  Readable after the failed launch (pinned host memory). */
int moco_p2p_last_timeout(uint32_t out[4]);

/* Cross-GPU stream-ordered barrier on peer-mapped signal pads (one uint32 slot
 * per writer rank on every rank): every rank stores `epoch` into slot[rank] of
 * every peer's pad (release, system scope), then waits until all `world` slots
 * of its own pad are >= epoch (acquire).  signal_pads_host: HOST array of `world`
 * device pointers to the pads (each >= world * 4 bytes, zero-initialised).
 * `epoch` must increase by 1 per event.  The wait is bounded in time (see moco_shuffle_gather_sync). */
int moco_signal_barrier(void* const* signal_pads_host, int world, int rank,
                        uint32_t epoch, void* stream);

/* ------------------------------------------------------------------------
 * Peer-memory plumbing for the two calls above (synchronous host functions;
 * the only entry points that allocate).  A buffer is cudaMalloc'ed and zeroed,
 * its 64-byte CUDA IPC handle is exchanged by the caller over its existing
 * process group (the reference's torch.distributed group, train.py:300), and
 * each peer maps it with moco_p2p_open (cudaIpcOpenMemHandle, lazy peer access).
 * ---------------------------------------------------------------------- */
int moco_p2p_alloc(size_t bytes, void** dev_ptr_out, unsigned char handle_out[64]);
int moco_p2p_open(const unsigned char handle[64], void** dev_ptr_out);
int moco_p2p_close(void* dev_ptr);
int moco_p2p_free(void* dev_ptr);

#ifdef __cplusplus
}
#endif
#endif /* MOCO_B200_H */
