"""One MoCo pretraining iteration -- the body of ``train_moco`` (train.py:244-283 of bl0/moco)
with the contrastive hot path on the sm_90a kernels.

Differences from the reference loop body, none of which change the math:
* the ShuffleBN image permute runs on a side stream, overlapped with the query-encoder forward;
* ``contrast.forward_loss`` replaces train.py:262-264 (logits never materialised) and contains the enqueue;
* no per-step ``.item()`` host syncs (train.py:280-281): loss / prob stay on the device;
* encoders run under bf16 autocast in channels_last (the reference used Apex AMP, train.py:189-196);
* with ``channels_last=True`` the two crops are taken straight from the 6-channel batch (train.py:250-254) as
  bf16 NHWC by one kernel each (x1: ``crop_to_channels_last_bf16``; x2: inside the ShuffleBN publish), which is
  what autocast + cuDNN would have produced with two more passes over the images; when the encoders' stem takes it
  (``encoders.StemConv``) the crops are written in the space-to-depth layout instead (``crop_to_s2d_bf16``), in which
  the 7x7 first convolution is a 16-channel 4x4 one -- for both crops on one GPU, for the query crop only when the
  key crops have to cross NVLink (``channels_last="nhwc"`` keeps the plain NHWC crops everywhere);
* ``fuse_normalize=True`` (SURVEY.md 8 f2): the encoders return their raw ``fc`` output and the L2 normalisation of
  ``moco/models/resnet.py:24-33`` -- forward for q, k and the enqueued keys, backward for q -- happens inside the
  head's two kernels instead of ~14 elementwise launches around them;
* ``graph_tail=True`` (single-GPU): everything after the key encoder (un-shuffle gather, head sweep, tail with the
  enqueue) is captured ONCE in a CUDA graph and replayed every step; the ring position lives on the device
  (``MemoryMoCo(device_index=True)``), which is what makes the replay correct.
"""
from __future__ import annotations

import torch

from .NCE import MemoryMoCo
from .NCE.Contrast import _nce_forward
from .util import DistributedShufle, _world, crop_to_channels_last_bf16, crop_to_s2d_bf16, moment_update, set_bn_train


def _unwrap(m):
    return m.module if hasattr(m, "module") else m


class MoCoStep:
    def __init__(self, model, model_ema, contrast: MemoryMoCo, optimizer, alpha: float = 0.999,
                 amp_dtype=torch.bfloat16, overlap_shuffle: bool = True, channels_last: bool = False,
                 fuse_normalize: bool = False, graph_tail: bool = False):
        self.model, self.model_ema, self.contrast, self.optimizer = model, model_ema, contrast, optimizer
        self.alpha = alpha
        self.amp_dtype = amp_dtype
        # fused input path only where it is value-preserving: bf16 autocast would round the images identically
        self.nhwc = bool(channels_last) and amp_dtype is torch.bfloat16
        # ... and in the space-to-depth layout when both stems take it (encoders.StemConv): channels_last="nhwc" keeps
        # the plain 3-channel NHWC crops
        self.s2d = (self.nhwc and channels_last != "nhwc" and getattr(_unwrap(model), "accepts_s2d", False)
                    and getattr(model_ema, "accepts_s2d", False))
        self.side = torch.cuda.Stream() if overlap_shuffle else None
        self.fuse_normalize = bool(fuse_normalize)
        if self.fuse_normalize:
            if not isinstance(contrast, MemoryMoCo):
                raise ValueError("fuse_normalize needs a MemoryMoCo head")
            for enc in (_unwrap(model), model_ema):
                if not hasattr(enc, "l2norm"):
                    raise ValueError("fuse_normalize needs encoders with an `l2norm` switch (moco_b200.encoders)")
                enc.l2norm = False
        self.graph_tail = bool(graph_tail)
        if self.graph_tail:
            if _world()[1] != 1:
                raise ValueError("graph_tail: the cross-GPU signal barrier carries a per-call epoch argument; "
                                 "the captured tail is single-GPU only")
            if not isinstance(contrast, MemoryMoCo) or not contrast.device_index:
                raise ValueError("graph_tail needs MemoryMoCo(device_index=True): a replayed graph cannot see a host-side "
                                 "ring position")
        self._graph = None
        self._warm = 0
        self.model.train()
        set_bn_train(self.model_ema)                     # train.py:235-236

    # ---- everything after the key encoder, eager -------------------------------------------------------------
    def _tail_eager(self, feat_q, feat_k, backward_inds):
        feat_k_all, feat_k = DistributedShufle.backward_shuffle(feat_k, backward_inds, return_local=True)   # train.py:260
        if self.fuse_normalize:
            loss, prob = self.contrast.forward_loss(feat_q, feat_k, feat_k_all, normalize=True)
        else:
            loss, prob = self.contrast.forward_loss(feat_q, feat_k, feat_k_all)          # train.py:262-264
        self.optimizer.zero_grad(set_to_none=True)                                       # train.py:267-268
        loss.backward()                                                                  # train.py:273
        return loss, prob

    # ---- the same, captured once and replayed ----------------------------------------------------------------
    def _tail_graphed(self, feat_q, feat_k, backward_inds):
        c = self.contrast
        if self._warm < 1:                              # first step eager: one-time kernel attribute / descriptor set-up
            self._warm += 1
            return self._tail_eager(feat_q, feat_k, backward_inds)
        if self._graph is None or self._gq.shape != feat_q.shape or self._gk.shape != feat_k.shape:
            self._gq = torch.empty_like(feat_q.detach())
            self._gk = torch.empty_like(feat_k)
            self._ginds = backward_inds.clone()         # own storage: later epochs' permutations are copied into it
            self._ginds_src = backward_inds

            def body():
                k_all, k_loc = DistributedShufle.backward_shuffle(self._gk, self._ginds, return_local=True)
                _, loss_prob, dq, _, _ = _nce_forward(c, self._gq, k_loc, False, True, c.kernel_flags, k_all=k_all,
                                                      normalize=self.fuse_normalize)
                return loss_prob, dq
            c._queue_bf16()
            c._index_dev()
            self._gq.copy_(feat_q.detach())
            self._gk.copy_(feat_k)
            self._graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self._graph):
                self._gout = body()
            # the capture itself ran nothing; the Python-side bookkeeping it did (host index mirror) is undone
            c.index = (c.index - self._gk.shape[0]) % c.queue_size
            c._index_shadow = c.index
        elif backward_inds is not self._ginds_src:
            self._ginds.copy_(backward_inds)            # a new epoch's permutation, same storage
            self._ginds_src = backward_inds
        self._gq.copy_(feat_q.detach())
        self._gk.copy_(feat_k)
        self._graph.replay()
        n_all = self._gk.shape[0]
        c.index = (c.index + n_all) % c.queue_size      # host mirror of the device-side ring position
        c._index_shadow = c.index
        c._bf16_src = (c.memory.data_ptr(), c.memory._version)
        loss_prob, dq = self._gout
        self.optimizer.zero_grad(set_to_none=True)
        feat_q.backward(dq.to(feat_q.dtype))                                             # train.py:273
        return loss_prob[0], loss_prob[1]

    def __call__(self, x1: torch.Tensor, x2: torch.Tensor, epoch: int):
        """x1, x2: [N, 3, 224, 224] CUDA tensors (the two crops, train.py:250-254).
        Returns (loss, prob) as 0-d CUDA tensors."""
        main = torch.cuda.current_stream()
        # bf16 NHWC crops; in the space-to-depth layout when both encoders' stems take it and the images allow it
        layout = self.nhwc and ("s2d" if (self.s2d and x1.shape[1] == 3 and x1.shape[2] % 2 == 0 and x1.shape[3] % 2 == 0)
                                else True)
        # Key crops that cross NVLink stay plain bf16 NHWC rows (301 KB at 224 x 224): the space-to-depth rows are 423 KB,
        # a quarter of it zero channels, and measured at 8 GPUs they pull at 517 GB/s (0.57 of the link) against
        # 547-564 GB/s for the plain rows -- the key encoder's first convolution then runs on 3 channels.
        layout_k = True if (layout == "s2d" and _world()[1] > 1) else layout
        if self.side is not None:
            # ShuffleBN forward (train.py:258) on the side stream while the query encoder runs
            self.side.wait_stream(main)
            with torch.cuda.stream(self.side), torch.no_grad():
                x2_shuffled, backward_inds = DistributedShufle.forward_shuffle(x2, epoch, cast_dtype=self.amp_dtype,
                                                                               channels_last=layout_k)
            x2.record_stream(self.side)
        if self.nhwc:
            x1 = crop_to_s2d_bf16(x1) if layout == "s2d" else crop_to_channels_last_bf16(x1)
        with torch.autocast("cuda", dtype=self.amp_dtype, enabled=self.amp_dtype is not None):
            feat_q = self.model(x1)                                                  # train.py:256
        with torch.no_grad():
            if self.side is not None:
                main.wait_stream(self.side)
                x2_shuffled.record_stream(main)
            else:
                x2_shuffled, backward_inds = DistributedShufle.forward_shuffle(x2, epoch, cast_dtype=self.amp_dtype,
                                                                               channels_last=layout_k)
            with torch.autocast("cuda", dtype=self.amp_dtype, enabled=self.amp_dtype is not None):
                feat_k = self.model_ema(x2_shuffled)                                 # train.py:259
        if self.graph_tail:
            loss, prob = self._tail_graphed(feat_q, feat_k, backward_inds)
        else:
            loss, prob = self._tail_eager(feat_q, feat_k, backward_inds)
        self.optimizer.step()                                                        # train.py:274
        moment_update(_unwrap(self.model), self.model_ema, self.alpha)               # train.py:277
        return loss, prob
