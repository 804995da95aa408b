"""BatchNorm2d with the block's ReLU / residual add folded in, on this library's channels_last bf16 kernels.

The reference's encoders apply ``nn.BatchNorm2d`` -> [``out += residual``] -> [``nn.ReLU``] at
``moco/models/resnet.py:42-63,74-102,114,139-143,156-157``; ShuffleBN (``moco/util.py:69-93``) exists for exactly these
batch statistics, and left to ATen's channels_last kernels they take most of the GPU time of a step.  :class:`BatchNormAct2d` is an ``nn.BatchNorm2d`` (same parameters,
buffers and ``state_dict`` keys, same running-statistics updates) whose training-mode forward / backward on CUDA
bf16 channels_last activations are two launches each of ``csrc/bn_nhwc.cu`` (``moco_bn_fwd_train`` / ``moco_bn_bwd``).
A block's residual BatchNorm, ``relu(bn(x) + r)``, runs ``moco_bn_add_relu_*`` instead: the forward writes the ReLU
mask as bits for the backward rather than having it re-read ``y``, and in a downsample block (``forward(x, residual,
shortcut_bn=...)``) the shortcut's BatchNorm runs inside the same passes, so neither its output nor the gradient
between the two BatchNorms is ever written.  The stem's BatchNorm + ReLU and its max pool (``forward_maxpool``) run
as ``moco_bn_relu_maxpool_fwd_train``: the pool applies the BatchNorm to each tap, so the stem's full-resolution
activation is never written.
The results are bit-identical to the separate calls.
Everything else -- CPU tensors, eval mode, fp32 or NCHW activations, channel counts the kernels do not take -- runs
``nn.BatchNorm2d``'s own forward followed by the add and the ReLU, i.e. exactly what the reference does.
"""
from __future__ import annotations

import torch
from torch import nn
import torch.nn.functional as F

from . import _lib

_workspaces = {}
_enabled = True
# bench.py's live roofline pass: a list makes every fused call append (kind, algorithmic bytes, start event, end event)
_prof = None


def _timed(kind, nbytes, call):
    if _prof is None:
        return call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    rc = call()
    e1.record()
    _prof.append((kind, nbytes, e0, e1))
    return rc


def set_fused(flag: bool) -> None:
    """Process-wide switch (A/B timing, debugging): False sends every BatchNormAct2d through the torch ops."""
    global _enabled
    _enabled = bool(flag)


def _workspace(device):
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    ws = _workspaces.get(key)
    if ws is None:
        ws = torch.zeros(_lib.load().moco_bn_workspace_bytes(), dtype=torch.uint8, device=device)   # zeroed once
        _workspaces[key] = ws
    return ws


def _rows_ok(t, like=None):
    return (t.is_cuda and t.dtype == torch.bfloat16 and t.dim() == 4 and t.numel() > 0
            and t.is_contiguous(memory_format=torch.channels_last) and (like is None or t.shape == like.shape))


class _BatchNormActFn(torch.autograd.Function):
    """y = relu?(batch_norm_train(x) [+ residual]); x, residual, y bf16 channels_last; weight / bias fp32."""

    @staticmethod
    def forward(ctx, x, weight, bias, residual, running_mean, running_var, num_batches_tracked, momentum, eps, relu):
        lib = _lib.load()
        N, C, H, W = x.shape
        M = N * H * W
        y = torch.empty_like(x)                                   # keeps the channels_last strides
        mean = torch.empty(C, dtype=torch.float32, device=x.device)
        invstd = torch.empty_like(mean)
        ws = _workspace(x.device)
        # algorithmic bytes: statistics read x; apply reads x (+ residual) and writes y
        code = _timed("bn_fwd", M * C * 2 * (3 + (residual is not None)), lambda: lib.moco_bn_fwd_train(
            x.data_ptr(), residual.data_ptr() if residual is not None else None, y.data_ptr(), M, C,
            weight.data_ptr(), bias.data_ptr(),
            running_mean.data_ptr() if running_mean is not None else None,
            running_var.data_ptr() if running_var is not None else None,
            num_batches_tracked.data_ptr() if num_batches_tracked is not None else None,
            float(momentum), float(eps), int(relu), mean.data_ptr(), invstd.data_ptr(), ws.data_ptr(), ws.numel(),
            _lib.cur_stream()))
        _lib.check(code, "moco_bn_fwd_train")
        ctx.relu = bool(relu)
        ctx.has_res = residual is not None
        # the ReLU mask of the backward is recomputed from x unless a residual went into it
        ctx.save_for_backward(x, y if (relu and residual is not None) else None, weight, bias, mean, invstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y, weight, bias, mean, invstd = ctx.saved_tensors
        lib = _lib.load()
        N, C, H, W = x.shape
        if dy.dtype != torch.bfloat16:
            dy = dy.to(torch.bfloat16)
        dy = dy.contiguous(memory_format=torch.channels_last)
        dx = torch.empty_like(x)
        want_res = ctx.has_res and ctx.needs_input_grad[3]
        if want_res and not ctx.relu:
            dres, dres_ptr = dy, None                             # without a ReLU the residual's gradient is dy itself
        elif want_res:
            dres = torch.empty_like(x)
            dres_ptr = dres.data_ptr()
        else:
            dres, dres_ptr = None, None
        dgamma = torch.empty(C, dtype=torch.float32, device=x.device)
        dbeta = torch.empty_like(dgamma)
        ws = _workspace(x.device)
        # algorithmic bytes: reduce reads dy, x (+ y for the mask); apply reads the same and writes dx (+ d residual)
        ops = 2 * (2 + (y is not None)) + 1 + (dres_ptr is not None)
        code = _timed("bn_bwd", N * H * W * C * 2 * ops, lambda: lib.moco_bn_bwd(
            dy.data_ptr(), x.data_ptr(), y.data_ptr() if y is not None else None, N * H * W, C,
            weight.data_ptr(), bias.data_ptr(), mean.data_ptr(), invstd.data_ptr(), int(ctx.relu),
            int(ctx.has_res), dx.data_ptr(), dres_ptr, dgamma.data_ptr(), dbeta.data_ptr(),
            ws.data_ptr(), ws.numel(), _lib.cur_stream()))
        _lib.check(code, "moco_bn_bwd")
        return dx, dgamma, dbeta, dres, None, None, None, None, None, None


def _layer(weight, bias, mean, invstd, stats=None, dgamma=None, dbeta=None):
    """moco_bn_layer of one BatchNorm: stats = (running_mean, running_var, num_batches_tracked, momentum, eps)."""
    ptr = lambda t: t.data_ptr() if t is not None else None
    rm, rv, nbt, momentum, eps = stats if stats is not None else (None, None, None, 0.0, 0.0)
    return _lib.BnLayer(ptr(weight), ptr(bias), ptr(rm), ptr(rv), ptr(nbt), float(momentum), float(eps), ptr(mean),
                        ptr(invstd), ptr(dgamma), ptr(dbeta))


class _BatchNormAddReluFn(torch.autograd.Function):
    """y = relu(batch_norm_train(x) + r); r = residual, or with a shortcut BN r = bf16(shortcut_bn(residual)) where
    residual is the shortcut convolution's raw output (a downsample block).  The backward reads the ReLU mask as bits
    written by the forward instead of y; the shortcut BN's output and the gradient between the two BNs are never
    materialised.  Same values as _BatchNormActFn (+ the shortcut BN's own pass)."""

    @staticmethod
    def forward(ctx, x, residual, weight, bias, sc_weight, sc_bias, stats, sc_stats, want_mask):
        lib = _lib.load()
        N, C, H, W = x.shape
        M = N * H * W
        y = torch.empty_like(x)
        mask = torch.empty((M, C // 8), dtype=torch.uint8, device=x.device) if want_mask else None
        f32 = lambda: torch.empty(C, dtype=torch.float32, device=x.device)
        mean, invstd = f32(), f32()
        bn = _layer(weight, bias, mean, invstd, stats)
        sc, sc_mean, sc_invstd = None, None, None
        if sc_weight is not None:
            sc_mean, sc_invstd = f32(), f32()
            sc = _layer(sc_weight, sc_bias, sc_mean, sc_invstd, sc_stats)
        ws = _workspace(x.device)
        # algorithmic bytes: statistics read x (+ the shortcut input); apply reads x and residual, writes y (+ mask bits)
        nbytes = M * C * 2 * (4 + (sc is not None)) + (M * C // 8 if want_mask else 0)
        code = _timed("bn_fwd", nbytes, lambda: lib.moco_bn_add_relu_fwd_train(
            x.data_ptr(), residual.data_ptr(), y.data_ptr(), mask.data_ptr() if mask is not None else None, M, C, bn, sc,
            ws.data_ptr(), ws.numel(), _lib.cur_stream()))
        _lib.check(code, "moco_bn_add_relu_fwd_train")
        ctx.save_for_backward(x, residual if sc is not None else None, mask, weight, mean, invstd, sc_weight, sc_mean,
                              sc_invstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, residual, mask, weight, mean, invstd, sc_weight, sc_mean, sc_invstd = ctx.saved_tensors
        if mask is None:
            raise RuntimeError("moco_b200: BatchNormAct2d ran its forward without the ReLU mask (no input required grad)")
        lib = _lib.load()
        N, C, H, W = x.shape
        M = N * H * W
        if dy.dtype != torch.bfloat16:
            dy = dy.to(torch.bfloat16)
        dy = dy.contiguous(memory_format=torch.channels_last)
        dx = torch.empty_like(x)
        f32 = lambda: torch.empty(C, dtype=torch.float32, device=x.device)
        dgamma, dbeta = f32(), f32()
        bn = _layer(weight, None, mean, invstd, dgamma=dgamma, dbeta=dbeta)
        sc, sc_dgamma, sc_dbeta = None, None, None
        if sc_weight is not None:
            sc_dgamma, sc_dbeta = f32(), f32()
            sc = _layer(sc_weight, None, sc_mean, sc_invstd, dgamma=sc_dgamma, dbeta=sc_dbeta)
            dres = torch.empty_like(x)
        else:
            dres = torch.empty_like(x) if ctx.needs_input_grad[1] else None
        ws = _workspace(x.device)
        # algorithmic bytes: reduce reads dy, x, mask (+ shortcut input); apply reads the same and writes dx (+ d residual)
        nbytes = M * C * 2 * (5 + (dres is not None) + 2 * (sc is not None)) + 2 * (M * C // 8)
        code = _timed("bn_bwd", nbytes, lambda: lib.moco_bn_add_relu_bwd(
            dy.data_ptr(), x.data_ptr(), residual.data_ptr() if residual is not None else None, mask.data_ptr(), M, C,
            bn, sc, dx.data_ptr(), dres.data_ptr() if dres is not None else None, ws.data_ptr(), ws.numel(),
            _lib.cur_stream()))
        _lib.check(code, "moco_bn_add_relu_bwd")
        return dx, dres, dgamma, dbeta, sc_dgamma, sc_dbeta, None, None, None


class _BatchNormReluMaxPoolFn(torch.autograd.Function):
    """maxpool3x3s2(relu(batch_norm_train(x))) without writing the BatchNorm's output: the pool pass takes each tap
    through the BatchNorm + ReLU.  The backward is the pool's backward followed by the BatchNorm's (mask from x).  Same
    values as _BatchNormActFn followed by _MaxPool3x3s2Fn."""

    @staticmethod
    def forward(ctx, x, weight, bias, stats):
        lib = _lib.load()
        N, C, H, W = x.shape
        OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        y = torch.empty((N, C, OH, OW), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        taps = torch.empty((N, OH, OW, C), dtype=torch.uint8, device=x.device)
        mean = torch.empty(C, dtype=torch.float32, device=x.device)
        invstd = torch.empty_like(mean)
        bn = _layer(weight, bias, mean, invstd, stats)
        ws = _workspace(x.device)
        # algorithmic bytes: statistics read x; the pool pass reads x, writes y and the tap bytes
        nbytes = N * H * W * C * 2 * 2 + N * OH * OW * C * 3
        code = _timed("bn_fwd", nbytes, lambda: lib.moco_bn_relu_maxpool_fwd_train(
            x.data_ptr(), y.data_ptr(), taps.data_ptr(), N, H, W, C, bn, ws.data_ptr(), ws.numel(), _lib.cur_stream()))
        _lib.check(code, "moco_bn_relu_maxpool_fwd_train")
        ctx.save_for_backward(x, taps, weight, bias, mean, invstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, taps, weight, bias, mean, invstd = ctx.saved_tensors
        lib = _lib.load()
        N, C, H, W = x.shape
        if dy.dtype != torch.bfloat16:
            dy = dy.to(torch.bfloat16)
        dy = dy.contiguous(memory_format=torch.channels_last)
        # Rebuilding the pool's input gradient inside the BatchNorm's two passes (a <= 4-window gather per element)
        # measured slower than writing it once and streaming it: the pool's backward, then the BatchNorm's.
        g = torch.empty_like(x)
        _lib.check(lib.moco_maxpool3x3s2_bwd(dy.data_ptr(), taps.data_ptr(), g.data_ptr(), N, H, W, C, _lib.cur_stream()),
                   "moco_maxpool3x3s2_bwd")
        dx = torch.empty_like(x)
        dgamma = torch.empty(C, dtype=torch.float32, device=x.device)
        dbeta = torch.empty_like(dgamma)
        ws = _workspace(x.device)
        # algorithmic bytes: reduce reads g, x; apply reads g, x and writes dx
        code = _timed("bn_bwd", N * H * W * C * 2 * 5, lambda: lib.moco_bn_bwd(
            g.data_ptr(), x.data_ptr(), None, N * H * W, C, weight.data_ptr(), bias.data_ptr(), mean.data_ptr(),
            invstd.data_ptr(), 1, 0, dx.data_ptr(), None, dgamma.data_ptr(), dbeta.data_ptr(), ws.data_ptr(),
            ws.numel(), _lib.cur_stream()))
        _lib.check(code, "moco_bn_bwd")
        return dx, dgamma, dbeta, None


class BatchNormAct2d(nn.BatchNorm2d):
    """``nn.BatchNorm2d`` + optional residual add + optional ReLU (``forward(x, residual=None)``)."""

    def __init__(self, num_features, relu=False, **kw):
        super().__init__(num_features, **kw)
        self.relu = bool(relu)

    def _fusable(self, x, residual):
        C = self.num_features
        return (_enabled and self.training and self.affine and self.momentum is not None
                and _rows_ok(x) and (residual is None or _rows_ok(residual, x))
                and 64 <= C <= 2048 and (C & (C - 1)) == 0 and x.shape[1] == C
                and x.numel() // C > 1                 # a single value per channel: nn.BatchNorm2d's own error
                and self.weight.dtype == torch.float32 and self.weight.is_cuda
                and (self.running_mean is None or self.running_mean.dtype == torch.float32))

    def _stats(self):
        return (self.running_mean, self.running_var, self.num_batches_tracked if self.track_running_stats else None,
                self.momentum, self.eps)

    def forward(self, x, residual=None, shortcut_bn=None):
        """``shortcut_bn``: a downsample block's shortcut BatchNorm (no ReLU); ``residual`` is then its input, the
        shortcut convolution's raw output, and ``y = relu?(bn(x) + shortcut_bn(residual))``."""
        if shortcut_bn is not None:
            if (self.relu and not shortcut_bn.relu and self._fusable(x, residual)
                    and shortcut_bn._fusable(residual, None)):
                return self._add_relu(x, residual, shortcut_bn)
            residual = shortcut_bn(residual)
        if self._fusable(x, residual):
            if self.relu and residual is not None:
                return self._add_relu(x, residual, None)
            return _BatchNormActFn.apply(x, self.weight, self.bias, residual, self.running_mean, self.running_var,
                                         self.num_batches_tracked if self.track_running_stats else None,
                                         self.momentum, self.eps, self.relu)
        y = super().forward(x)
        if residual is not None:
            y = y + residual
        return F.relu(y, inplace=True) if self.relu else y

    def forward_maxpool(self, x, pool):
        """``pool(self(x))`` for a :class:`MaxPool3x3s2` ``pool`` (the stem): one pass applies the BatchNorm + ReLU to
        every tap of the pool, so that the BatchNorm's output is never written."""
        if self.relu and isinstance(pool, MaxPool3x3s2) and self._fusable(x, None):
            return _BatchNormReluMaxPoolFn.apply(x, self.weight, self.bias, self._stats())
        return pool(self(x))

    def _add_relu(self, x, residual, sc):
        params = (x, residual, self.weight, self.bias) + ((sc.weight, sc.bias) if sc is not None else ())
        want_mask = torch.is_grad_enabled() and any(t.requires_grad for t in params)
        return _BatchNormAddReluFn.apply(x, residual, self.weight, self.bias,
                                         sc.weight if sc is not None else None, sc.bias if sc is not None else None,
                                         self._stats(), sc._stats() if sc is not None else None, want_mask)

    def extra_repr(self):
        return super().extra_repr() + f", relu={self.relu}"


class _MaxPool3x3s2Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        lib = _lib.load()
        N, C, H, W = x.shape
        OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        y = torch.empty((N, C, OH, OW), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        taps = torch.empty((N, OH, OW, C), dtype=torch.uint8, device=x.device)
        _lib.check(lib.moco_maxpool3x3s2_fwd(x.data_ptr(), y.data_ptr(), taps.data_ptr(), N, H, W, C, _lib.cur_stream()),
                   "moco_maxpool3x3s2_fwd")
        ctx.save_for_backward(taps)
        ctx.shape = (N, C, H, W)
        return y

    @staticmethod
    def backward(ctx, dy):
        (taps,) = ctx.saved_tensors
        N, C, H, W = ctx.shape
        if dy.dtype != torch.bfloat16:
            dy = dy.to(torch.bfloat16)
        dy = dy.contiguous(memory_format=torch.channels_last)
        dx = torch.empty((N, C, H, W), dtype=torch.bfloat16, device=dy.device, memory_format=torch.channels_last)
        _lib.check(_lib.load().moco_maxpool3x3s2_bwd(dy.data_ptr(), taps.data_ptr(), dx.data_ptr(), N, H, W, C,
                                                     _lib.cur_stream()), "moco_maxpool3x3s2_bwd")
        return dx


class MaxPool3x3s2(nn.MaxPool2d):
    """``nn.MaxPool2d(kernel_size=3, stride=2, padding=1)`` (moco/models/resnet.py:119): this library's kernels for CUDA
    bf16 channels_last activations, ``nn.MaxPool2d``'s own forward for anything else."""

    def __init__(self):
        super().__init__(kernel_size=3, stride=2, padding=1)

    def forward(self, x):
        if _enabled and _rows_ok(x) and x.shape[1] % 8 == 0:
            return _MaxPool3x3s2Fn.apply(x)
        return super().forward(x)
