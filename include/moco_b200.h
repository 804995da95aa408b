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
 *     cached cuTensorMapEncodeTiled entry point; they are CUDA-graph capturable;
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

#define MOCO_B200_ABI_VERSION 3 /* 3: + moco_bn_*, moco_maxpool3x3s2_*, moco_crop_s2d_bf16 (additive) */

enum {
    MOCO_OK = 0,
    MOCO_ERR_INVALID = -1,     /* bad argument (null pointer, size, alignment)          */
    MOCO_ERR_UNSUPPORTED = -2, /* valid but not implemented for this shape/dtype/device */
    MOCO_ERR_WORKSPACE = -3,   /* workspace too small                                    */
    MOCO_ERR_CUDA = -4         /* a CUDA runtime/driver call failed                      */
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
                               /* 6NCK, 2NK) plus ONE tail kernel: each (CTA, row) stabilises with the row   */
                               /* maximum of the CTA's first tile.  A row whose partial sum leaves the safe  */
                               /* range (a later logit > ~100 binades above that maximum: un-normalised      */
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
 * order, no float atomics).
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
 * Shapes outside the one-sweep envelope fall back to the moco_nce_fwd kernels
 * followed by the enqueue kernel (then normalize and index_dev must be 0/NULL:
 * MOCO_ERR_UNSUPPORTED otherwise).
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
 * Contrast.py:18).  Requires n_all <= K (SURVEY S10).
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
 * Same numerical contract as MOCO_NCE_ONE_PASS of moco_nce_fwd.
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
 * (mask recomputed from x when has_residual == 0, read from y otherwise -- y may be
 * NULL unless relu && has_residual):  dbeta = sum g,  dgamma = sum g * x^,
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
 * deterministic).  One launch each.
 * ---------------------------------------------------------------------- */
int moco_maxpool3x3s2_fwd(const void* x, void* y, void* taps_u8, int N, int H, int W, int C, void* stream);
int moco_maxpool3x3s2_bwd(const void* dy, const void* taps_u8, void* dx, int N, int H, int W, int C, void* stream);

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
