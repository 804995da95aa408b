"""MemoryMoCo -- the MoCo queue + InfoNCE head behind the reference's own API.

Mirrors ``moco/NCE/Contrast.py:6-36`` of bl0/moco (same constructor, attributes,
buffers, ``state_dict`` keys and ``forward(q, k, k_all) -> [N, K+1]`` contract) but
every device-side step is a hand-written sm_90a kernel reached through the C ABI
(``include/moco_b200.h``):

* ``forward_loss(q, k, k_all) -> (loss, prob)``: the fused fast path.  The
  q.Queue^T contraction, /T, log-sum-exp, cross-entropy, ``prob`` metric AND the
  gradient w.r.t. q are produced by tensor-core (wgmma) kernels before the enqueue; the
  [N, K+1] logits never reach HBM and the queue is never cloned.
* ``forward(q, k, k_all) -> out``: API-compatible dense logits (the kernel's
  epilogue writes them).  The returned tensor also carries the fused loss so that
  ``NCESoftmaxLoss`` (NCECriterion.py) does not have to re-read it.
"""
from __future__ import annotations

import math

import torch
from torch import nn

from .. import _lib


class _Scratch:
    """Per-(N, C, K, device) output + workspace buffers (allocated once; stable
    addresses keep the calls CUDA-graph capturable)."""

    def __init__(self, N, C, K, device):
        lib = _lib.load()
        f32 = dict(dtype=torch.float32, device=device)
        self.lse = torch.empty(N, **f32)
        self.loss_rows = torch.empty(N, **f32)
        self.prob_rows = torch.empty(N, **f32)
        self.ws_bytes = int(lib.moco_nce_workspace_bytes(N, C, K))
        self.ws = torch.empty(self.ws_bytes + 256, dtype=torch.uint8, device=device)
        off = (-self.ws.data_ptr()) % 256
        self.ws_ptr = self.ws.data_ptr() + off


def _aligned16(t):
    """The kernels read q and k_all with 16-byte vector loads (include/moco_b200.h): a contiguous view that starts at
    an odd storage offset is copied."""
    return t if t.data_ptr() % 16 == 0 else t.clone()


def _nce_forward(mod: "MemoryMoCo", q, k, want_logits: bool, want_dq: bool, flags: int, k_all=None,
                 normalize: bool = False):
    """One head evaluation.  With ``k_all`` the FIFO enqueue (Contrast.py:29-34) is part of the same C call
    (``moco_nce_step``: two kernels for loss, prob, dq and the enqueue) and the module's ring position is advanced."""
    lib = _lib.load()
    _lib.require_cuda(q, k, mod.memory)
    if q.dim() != 2 or q.shape != k.shape or q.shape[1] != mod.memory.shape[1]:
        raise ValueError(f"MemoryMoCo: q {tuple(q.shape)} / k {tuple(k.shape)} do not match the queue "
                         f"{tuple(mod.memory.shape)}")
    if q.device != mod.memory.device or k.device != mod.memory.device:
        raise RuntimeError(f"MemoryMoCo: q on {q.device}, k on {k.device}, queue on {mod.memory.device}")
    if q.dtype != k.dtype:
        k = k.to(q.dtype)
    q = _aligned16(q.contiguous())
    k = k.contiguous()
    N, C = q.shape
    K = mod.queue_size
    queue = mod._queue_bf16()
    key = (N, C, K, q.device)
    sc = mod._scratch.get(key)
    if sc is None:
        sc = mod._scratch[key] = _Scratch(N, C, K, q.device)
    logits = torch.empty(N, K + 1, dtype=torch.float32, device=q.device) if want_logits else None
    dq = torch.empty(N, C, dtype=torch.float32, device=q.device) if want_dq else None
    loss_prob = torch.empty(2, dtype=torch.float32, device=q.device)
    if k_all is None:
        if normalize:
            raise RuntimeError("MemoryMoCo: in-kernel normalisation is part of the fused step (k_all required)")
        code = lib.moco_nce_fwd(
            q.data_ptr(), k.data_ptr(), _lib.dtype_code(q), queue.data_ptr(), N, C, K,
            1.0 / mod.temperature,
            logits.data_ptr() if logits is not None else None,
            sc.lse.data_ptr(), sc.loss_rows.data_ptr(), sc.prob_rows.data_ptr(), loss_prob.data_ptr(),
            dq.data_ptr() if dq is not None else None,
            sc.ws_ptr, sc.ws_bytes, flags, _lib.cur_stream())
        _lib.check(code, "moco_nce_fwd")
    else:
        k_all = mod._check_keys(k_all)
        idx_dev = mod._index_dev()
        code = lib.moco_nce_step(
            q.data_ptr(), k.data_ptr(), _lib.dtype_code(q), 1 if normalize else 0, queue.data_ptr(),
            mod.memory.data_ptr(), N, C, K, 1.0 / mod.temperature, k_all.data_ptr(), _lib.dtype_code(k_all),
            k_all.shape[0], mod.index, idx_dev.data_ptr() if idx_dev is not None else None,
            sc.lse.data_ptr(), sc.loss_rows.data_ptr(), sc.prob_rows.data_ptr(), loss_prob.data_ptr(),
            dq.data_ptr() if dq is not None else None, sc.ws_ptr, sc.ws_bytes, flags, _lib.cur_stream())
        _lib.check(code, "moco_nce_step")
        mod._after_enqueue(k_all.shape[0])
    return logits, loss_prob, dq, q, k


class _FusedNCE(torch.autograd.Function):
    """(loss, prob) = InfoNCE(q, k, queue), then the enqueue of k_all -- one C call, two kernels.
    backward: grad_q = grad_loss * dq (dq comes out of the forward's kernels)."""

    @staticmethod
    def forward(ctx, q, k, k_all, mod, flags, normalize):
        need_dq = q.requires_grad
        ctx.set_materialize_grads(False)
        _, loss_prob, dq, _, _ = _nce_forward(mod, q.detach(), k.detach(), False, need_dq, flags, k_all=k_all.detach(),
                                              normalize=normalize)
        ctx.dq = dq
        ctx.q_dtype = q.dtype
        loss, prob = loss_prob[0], loss_prob[1]
        ctx.mark_non_differentiable(prob)
        return loss, prob

    @staticmethod
    def backward(ctx, g_loss, g_prob):
        dq = ctx.dq
        if dq is None or g_loss is None:
            return None, None, None, None, None, None
        return (dq * g_loss).to(ctx.q_dtype), None, None, None, None, None


class _FusedNCEWithLogits(torch.autograd.Function):
    """Dense-logits API: returns (out, loss, prob).  ``out`` has the dense backward
    (arbitrary upstream gradient); ``loss`` has the fused backward."""

    @staticmethod
    def forward(ctx, q, k, mod, flags):
        need = q.requires_grad
        # without this autograd hands backward() a zero-filled [N, K+1] gradient for `out` whenever only the
        # loss was back-propagated (the reference call site, train.py:262-273): 67 MB of zeros per step at
        # configs[2] plus a dense contraction over the whole queue, all to add 0
        ctx.set_materialize_grads(False)
        logits, loss_prob, dq, qc, kc = _nce_forward(mod, q.detach(), k.detach(), True, need, flags)
        ctx.dq = dq
        ctx.q_dtype = q.dtype
        ctx.inv_T = 1.0 / mod.temperature
        ctx.K = mod.queue_size
        if need:
            # The dense backward (a gradient arriving through `out` itself) needs the PRE-enqueue rows.  The
            # reference clones the whole queue every step for that (Contrast.py:25); here only the <= all_size rows
            # the coming enqueue overwrites are stashed -- by MemoryMoCo.forward, right before it enqueues -- and
            # the backward patches them back into a copy only if that gradient really arrives.
            ctx.save_for_backward(kc)
            ctx.mod = mod
            ctx.stash = None                       # (ring index, rows [n, C] bf16) set by MemoryMoCo.forward
            mod._pending_dense_ctx = ctx
        loss, prob = loss_prob[0], loss_prob[1]
        ctx.mark_non_differentiable(prob)
        return logits, loss, prob

    @staticmethod
    def backward(ctx, g_out, g_loss, g_prob):
        if ctx.dq is None:
            return None, None, None, None
        grad = None
        if g_loss is not None:
            grad = ctx.dq * g_loss
        if g_out is not None:
            (kc,) = ctx.saved_tensors
            queue_pre = ctx.mod._queue_bf16()
            if ctx.stash is not None:              # rebuild the snapshot the forward saw
                if ctx.mod._enqueue_count != ctx.stash[2] + 1:
                    raise RuntimeError("MemoryMoCo: backward through the dense logits after a later step already "
                                       "enqueued into the queue; call backward() before the next forward()")
                queue_pre = queue_pre.clone()
                idx0, rows = ctx.stash[0], ctx.stash[1]
                ids = (torch.arange(rows.shape[0], device=rows.device) + idx0) % ctx.K
                queue_pre[ids] = rows
            lib = _lib.load()
            g = g_out.contiguous().float()
            N, C = kc.shape
            dq2 = torch.empty(N, C, dtype=torch.float32, device=g.device)
            code = lib.moco_nce_bwd_dense(g.data_ptr(), kc.data_ptr(), _lib.dtype_code(kc), queue_pre.data_ptr(),
                                          N, C, ctx.K, ctx.inv_T, dq2.data_ptr(), _lib.cur_stream())
            _lib.check(code, "moco_nce_bwd_dense")
            grad = dq2 if grad is None else grad + dq2
        return (grad.to(ctx.q_dtype) if grad is not None else None), None, None, None


class MemoryMoCo(nn.Module):
    """Fixed-size queue with momentum encoder (drop-in for moco.NCE.MemoryMoCo)."""

    def __init__(self, feature_dim, queue_size, temperature=0.07, persist_index=False, device_index=False):
        super().__init__()
        self.queue_size = queue_size
        # device_index=True keeps a device copy of the ring position that the kernels advance (CUDA-graph replay)
        self.device_index = bool(device_index)
        self._index_t = None
        self._index_shadow = 0
        self.temperature = temperature
        self.index = 0
        self.kernel_flags = _lib.NCE_AUTO
        # The reference never checkpoints `index` (Contrast.py:12; train.py:145,163), so a resumed run restarts
        # the ring at slot 0.  persist_index=True (extension, SURVEY.md §8 f4) parks the write position in the
        # otherwise vestigial `params` buffer: same state_dict keys/shapes, the reference ignores the value, and
        # a reference checkpoint (params == -1) still loads with index 0.  Off by default = reference behaviour.
        self.persist_index = bool(persist_index)

        # same buffers / init / state_dict keys as the reference (Contrast.py:15-18)
        self.register_buffer('params', torch.tensor([-1]))
        stdv = 1. / math.sqrt(feature_dim / 3)
        memory = torch.rand(self.queue_size, feature_dim, requires_grad=False).mul_(2 * stdv).add_(-stdv)
        self.register_buffer('memory', memory)
        # bf16 working copy read by the tensor-core kernels; rebuilt from `memory` on demand
        self.register_buffer('memory_bf16', torch.empty(0, dtype=torch.bfloat16), persistent=False)
        self._bf16_src = None      # (data_ptr, _version) of `memory` the bf16 copy was built from
        self._scratch = {}
        self._enqueue_count = 0
        self._pending_dense_ctx = None
        self.register_load_state_dict_post_hook(lambda m, keys: m._after_load())

    # -- checkpoint format (train.py:145,163): keys {'params', 'memory'}, fp32 [K, C] ------------------
    def _save_to_state_dict(self, destination, prefix, keep_vars):
        if self.persist_index:
            if self.device_index:
                self.sync_index()                         # graph replays advance only the device copy
            self.params.fill_(int(self.index))
        super()._save_to_state_dict(destination, prefix, keep_vars)

    def _after_load(self):
        self._invalidate()
        self._index_t = None
        if self.persist_index:
            saved = int(self.params.item())
            self.index = saved % self.queue_size if saved >= 0 else 0

    # -- bf16 working queue -------------------------------------------------
    def _invalidate(self):
        self._bf16_src = None

    def _apply(self, fn, *a, **kw):      # .cuda() / .to(): buffers move, caches die
        out = super()._apply(fn, *a, **kw)
        self._invalidate()
        self._scratch = {}
        self._index_t = None
        return out

    def _check_buffers(self):
        """The C ABI takes raw pointers: `memory` must be exactly the fp32 row-major [K, C] buffer the kernels
        index (module.half() / .double() / .to(dtype) convert registered buffers behind our back)."""
        mem = self.memory
        if mem.dtype != torch.float32 or not mem.is_contiguous() or mem.dim() != 2 or mem.shape[0] != self.queue_size:
            raise RuntimeError(f"MemoryMoCo: `memory` must stay a contiguous float32 [queue_size, C] buffer "
                               f"(got {mem.dtype}, shape {tuple(mem.shape)}); keep the module in fp32 -- the kernels "
                               "maintain their own bf16 working copy")

    def _queue_bf16(self) -> torch.Tensor:
        mem = self.memory
        _lib.require_cuda(mem)
        self._check_buffers()
        tag = (mem.data_ptr(), mem._version)
        if self._bf16_src != tag or self.memory_bf16.shape != mem.shape or self.memory_bf16.device != mem.device:
            if self.memory_bf16.shape != mem.shape or self.memory_bf16.device != mem.device:
                self.memory_bf16 = torch.empty_like(mem, dtype=torch.bfloat16)
            lib = _lib.load()
            _lib.check(lib.moco_f32_to_bf16(mem.data_ptr(), self.memory_bf16.data_ptr(), mem.numel(),
                                            _lib.cur_stream()), "moco_f32_to_bf16")
            self._bf16_src = tag
        return self.memory_bf16

    # -- enqueue (Contrast.py:29-34) ----------------------------------------
    def _check_keys(self, k_all):
        _lib.require_cuda(k_all)
        k_all = _aligned16(k_all.detach().contiguous())
        if k_all.dim() != 2 or k_all.shape[1] != self.memory.shape[1]:
            raise ValueError(f"MemoryMoCo: k_all {tuple(k_all.shape)} does not match the queue "
                             f"{tuple(self.memory.shape)}")
        if k_all.device != self.memory.device:
            raise RuntimeError(f"MemoryMoCo: k_all on {k_all.device}, queue on {self.memory.device}")
        return k_all

    def _index_dev(self):
        """Device copy of the ring position (``device_index=True``): the kernels read it and advance it themselves,
        so a CUDA graph that captured the step replays correctly (the Python ``index`` stays a host mirror)."""
        if not self.device_index:
            return None
        if self._index_t is None or self._index_t.device != self.memory.device:
            self._index_t = torch.tensor([int(self.index)], dtype=torch.int64, device=self.memory.device)
        elif self._index_shadow != self.index:            # somebody assigned `index` on the host
            self._index_t.fill_(int(self.index))
        self._index_shadow = self.index
        return self._index_t

    def sync_index(self):
        """Refresh the host mirror ``index`` from the device copy (after CUDA-graph replays)."""
        if self._index_t is not None:
            self.index = int(self._index_t.item())
        return self.index

    def _after_enqueue(self, all_size):
        # the kernel wrote both copies; keep the cache tag in sync without bumping `memory._version`
        self._bf16_src = (self.memory.data_ptr(), self.memory._version)
        self.index = (self.index + all_size) % self.queue_size
        self._index_shadow = self.index                   # the fused step advanced the device copy too
        self._enqueue_count += 1

    @torch.no_grad()
    def enqueue(self, k_all):
        lib = _lib.load()
        k_all = self._check_keys(k_all)
        all_size, C = k_all.shape
        if self._index_t is not None and self.device_index:
            self._index_t.fill_(int(self.index))          # stand-alone enqueue: host index is the source of truth
        queue = self._queue_bf16()
        code = lib.moco_queue_enqueue(queue.data_ptr(), self.memory.data_ptr(), k_all.data_ptr(),
                                      _lib.dtype_code(k_all), all_size, C, self.queue_size, self.index,
                                      _lib.cur_stream())
        _lib.check(code, "moco_queue_enqueue")
        self._after_enqueue(all_size)
        if self._index_t is not None and self.device_index:
            self._index_t.fill_(int(self.index))

    # -- public API ----------------------------------------------------------
    def _can_fuse_normalize(self, q) -> bool:
        flags = self.kernel_flags
        return (q.requires_grad and q.shape[1] in (64, 128) and not (flags & (_lib.NCE_TWO_PASS | _lib.NCE_FORCE_SIMT))
                and ((flags & _lib.NCE_ONE_PASS) or 1.0 / self.temperature <= _lib.ONE_PASS_MAX_INV_T))

    def forward_loss(self, q, k, k_all, normalize=False):
        """Fused path: returns (loss, prob) == (NCESoftmaxLoss()(out), softmax(out,1)[:,0].mean())
        of the reference's train.py:262-264 and enqueues k_all -- two kernels in all (``moco_nce_step``).

        normalize=True: q, k, k_all are the encoders' RAW fc outputs; the rows are L2-normalised inside the kernels
        exactly like the reference's ``Normalize`` layer (moco/models/resnet.py:24-33) and the gradient that flows
        back is w.r.t. the raw q (SURVEY.md 8 f2).  Shapes the kernels do not fuse are normalised here in torch."""
        if normalize and not self._can_fuse_normalize(q):
            q = q / q.pow(2).sum(1, keepdim=True).pow(0.5)
            k = k / k.pow(2).sum(1, keepdim=True).pow(0.5)
            k_all = k_all / k_all.pow(2).sum(1, keepdim=True).pow(0.5)
            normalize = False
        return _FusedNCE.apply(q, k.detach(), k_all.detach(), self, self.kernel_flags, bool(normalize))

    def forward(self, q, k, k_all):
        out, loss, prob = _FusedNCEWithLogits.apply(q, k.detach(), self, self.kernel_flags)
        ctx, self._pending_dense_ctx = self._pending_dense_ctx, None
        if ctx is not None:
            # stash the rows this enqueue is about to overwrite (<= all_size x C bf16, e.g. 0.5 MB at configs[2])
            # instead of cloning the whole queue (Contrast.py:25) for a backward that usually never comes
            n = min(int(k_all.shape[0]), self.queue_size)
            ids = (torch.arange(n, device=self.memory.device) + self.index) % self.queue_size
            ctx.stash = (self.index, self._queue_bf16()[ids], self._enqueue_count)
        self.enqueue(k_all)
        # let NCESoftmaxLoss pick up the fused result instead of re-reading [N, K+1] logits
        out._moco_fused = (loss, prob, out._version)
        return out
