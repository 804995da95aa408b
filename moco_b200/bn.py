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
A block's input has two consumers; ``hand_over`` (called by the encoders' blocks in front of the residual branch)
passes that branch's gradient to the producer's backward, which adds it to the other one inside its own kernels
(``moco_bn_add_relu_bwd2`` / ``moco_maxpool3x3s2_bwd2``) instead of autograd adding them in a pass of its own.
The results are bit-identical to the separate calls.
A FROZEN module (``frozen = True``, set by :meth:`moco_b200.encoders.MoCoResNet.freeze`) in eval mode under
``torch.no_grad()`` -- the linear probe's encoder -- runs the eval kernels instead: the running statistics are folded
into a per-channel scale / shift (re-folded whenever the weights or statistics change), and one launch applies the
BatchNorm, the add (a downsample block's shortcut BatchNorm included) and the ReLU (``moco_bn_eval_act``), or also
the stem's max pool (``moco_bn_relu_maxpool_eval``) or the global average pool (``forward(..., avgpool=True)``,
``moco_bn_eval_act_avgpool``).  Their arithmetic is the header's eval contract, which separate fp32 torch ops
reproduce bit for bit.
Everything else -- CPU tensors, eval mode of a module that is not frozen, fp32 or NCHW activations, channel counts the
kernels do not take -- runs ``nn.BatchNorm2d``'s own forward followed by the add and the ReLU, i.e. exactly what the
reference does.
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


def _workspace(device, conv=False):
    """The stream's workspace of the BatchNorm entry points, or (conv=True) of moco_conv1x1_bn_stats."""
    key = (device.index, torch._C._cuda_getCurrentRawStream(device.index), conv)   # as _lib.cur_stream
    ws = _workspaces.get(key)
    if ws is None:
        lib = _lib.load()
        nbytes = lib.moco_conv1x1_workspace_bytes() if conv else lib.moco_bn_workspace_bytes()
        ws = torch.zeros(nbytes, dtype=torch.uint8, device=device)   # zeroed once
        _workspaces[key] = ws
    return ws


def _rows_ok(t, like=None):
    return (t.is_cuda and t.dtype == torch.bfloat16 and t.dim() == 4 and t.numel() > 0
            and t.is_contiguous(memory_format=torch.channels_last) and (like is None or t.shape == like.shape))


def _grad_rows(g):
    if g.dtype != torch.bfloat16:
        g = g.to(torch.bfloat16)
    return g.contiguous(memory_format=torch.channels_last)


def _take_handed(ctx):
    """The gradient a :class:`_HandOverFn` left on this node during the current backward (None without one), taken
    exactly once, so that a second backward through a retained graph sees only what its own hand-over leaves."""
    g = getattr(ctx, "handed", None)
    if g is None:
        return None
    ctx.handed = None
    return _grad_rows(g)


class _BatchNormActFn(torch.autograd.Function):
    """y = relu?(batch_norm_train(x) [+ residual]); x, residual, y bf16 channels_last; weight / bias fp32."""

    @staticmethod
    def forward(ctx, x, weight, bias, residual, running_mean, running_var, num_batches_tracked, momentum, eps, relu,
                given=None):
        """given: (mean, invstd) already computed by the producing convolution (:func:`conv1x1_stats`), which also
        updated the running statistics: only the apply pass runs."""
        lib = _lib.load()
        N, C, H, W = x.shape
        M = N * H * W
        y = torch.empty_like(x)                                   # keeps the channels_last strides
        ptr = lambda t: t.data_ptr() if t is not None else None
        if given is not None:
            mean, invstd = given
            bn = _layer(weight, bias, mean, invstd, (running_mean, running_var, num_batches_tracked, momentum, eps))
            # algorithmic bytes: apply reads x (+ residual) and writes y
            code = _timed("bn_fwd", M * C * 2 * (2 + (residual is not None)), lambda: lib.moco_bn_fwd_train_given(
                x.data_ptr(), ptr(residual), y.data_ptr(), None, M, C, int(relu), bn, None, _lib.BN_STATS_GIVEN,
                None, 0, _lib.cur_stream()))
            _lib.check(code, "moco_bn_fwd_train_given")
        else:
            mean = torch.empty(C, dtype=torch.float32, device=x.device)
            invstd = torch.empty_like(mean)
            ws = _workspace(x.device)
            # algorithmic bytes: statistics read x; apply reads x (+ residual) and writes y
            code = _timed("bn_fwd", M * C * 2 * (3 + (residual is not None)), lambda: lib.moco_bn_fwd_train(
                x.data_ptr(), ptr(residual), y.data_ptr(), M, C, weight.data_ptr(), bias.data_ptr(),
                ptr(running_mean), ptr(running_var), ptr(num_batches_tracked),
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
        return dx, dgamma, dbeta, dres, None, None, None, None, None, None, None


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
    def forward(ctx, x, residual, weight, bias, sc_weight, sc_bias, stats, sc_stats, want_mask, given=None,
                sc_given=None, recompute=None):
        """given / sc_given: (mean, invstd) of the BatchNorm / the shortcut BN already computed by the producing
        convolution (:func:`conv1x1_stats`), which also updated its running statistics; that statistics pass is
        skipped.  recompute: (a, w) with x = conv2d(a, w) of a 1x1 convolution (given required): y is computed from a
        by moco_conv1x1_bn_add_relu_fwd instead of reading x (:func:`conv1x1_bn_add_relu`)."""
        lib = _lib.load()
        N, C, H, W = x.shape
        M = N * H * W
        y = torch.empty_like(x)
        mask = torch.empty((M, C // 8), dtype=torch.uint8, device=x.device) if want_mask else None
        f32 = lambda: torch.empty(C, dtype=torch.float32, device=x.device)
        mean, invstd = given if given is not None else (f32(), f32())
        bn = _layer(weight, bias, mean, invstd, stats)
        sc, sc_mean, sc_invstd = None, None, None
        if sc_weight is not None:
            sc_mean, sc_invstd = sc_given if sc_given is not None else (f32(), f32())
            sc = _layer(sc_weight, sc_bias, sc_mean, sc_invstd, sc_stats)
        ws = _workspace(x.device)
        flags = (_lib.BN_STATS_GIVEN if given is not None else 0) | (_lib.BN_SC_STATS_GIVEN if sc_given is not None else 0)
        # algorithmic bytes: statistics read x (+ the shortcut input) unless given; apply reads x and residual, writes
        # y (+ mask bits)
        passes = (given is None) + (sc is not None and sc_given is None)
        nbytes = M * C * 2 * (3 + passes) + (M * C // 8 if want_mask else 0)
        mask_ptr = mask.data_ptr() if mask is not None else None
        if recompute is not None:
            a, w = recompute
            Cin = a.shape[1]
            # algorithmic bytes: reads a, residual (+ the shortcut input for its statistics), writes y (+ mask bits)
            nbytes = M * 2 * (Cin + C * (2 + passes)) + (M * C // 8 if want_mask else 0)
            code = _timed("bn_fwd", nbytes, lambda: lib.moco_conv1x1_bn_add_relu_fwd(
                a.data_ptr(), w.data_ptr(), residual.data_ptr(), y.data_ptr(), mask_ptr, M, Cin, C, bn, sc, flags,
                ws.data_ptr(), ws.numel(), _lib.cur_stream()))
            _lib.check(code, "moco_conv1x1_bn_add_relu_fwd")
        elif flags:
            code = _timed("bn_fwd", nbytes, lambda: lib.moco_bn_fwd_train_given(
                x.data_ptr(), residual.data_ptr(), y.data_ptr(), mask_ptr, M, C, 1, bn, sc, flags, ws.data_ptr(),
                ws.numel(), _lib.cur_stream()))
            _lib.check(code, "moco_bn_fwd_train_given")
        else:
            code = _timed("bn_fwd", nbytes, lambda: lib.moco_bn_add_relu_fwd_train(
                x.data_ptr(), residual.data_ptr(), y.data_ptr(), mask_ptr, M, C, bn, sc, ws.data_ptr(), ws.numel(),
                _lib.cur_stream()))
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
        dy = _grad_rows(dy)
        dx = torch.empty_like(x)
        reduced, ctx.reduced = getattr(ctx, "reduced", None), None
        if reduced is not None and dy.data_ptr() == reduced[0].data_ptr():
            # the consumer's dgrad formed g = dy and the sums (_dgrad_bn_bwd); another consumer adding to the gradient
            # gives a different tensor, which takes the full backward below (g is already masked: mask(g + e) = g +
            # mask(e))
            g, dgamma, dbeta = reduced
            bn = _layer(weight, None, mean, invstd, dgamma=dgamma, dbeta=dbeta)
            # algorithmic bytes: reads g and x, writes dx
            code = _timed("bn_bwd", M * C * 2 * 3, lambda: lib.moco_bn_bwd_apply_given(
                g.data_ptr(), x.data_ptr(), None, M, C, bn, None, dx.data_ptr(), None, _lib.cur_stream()))
            _lib.check(code, "moco_bn_bwd_apply_given")
            return (dx, g if ctx.needs_input_grad[1] else None, dgamma, dbeta, None, None, None, None, None, None, None,
                    None)
        dy2 = _take_handed(ctx)          # y's other consumer's gradient: summed inside both passes
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
        # algorithmic bytes: reduce reads dy (+ dy2), x, mask (+ shortcut input); apply reads the same and writes dx
        # (+ d residual)
        nbytes = (M * C * 2 * (5 + (dres is not None) + 2 * (sc is not None) + 2 * (dy2 is not None))
                  + 2 * (M * C // 8))
        ptr = lambda t: t.data_ptr() if t is not None else None
        if dy2 is None:
            code = _timed("bn_bwd", nbytes, lambda: lib.moco_bn_add_relu_bwd(
                dy.data_ptr(), x.data_ptr(), ptr(residual), mask.data_ptr(), M, C, bn, sc, dx.data_ptr(), ptr(dres),
                ws.data_ptr(), ws.numel(), _lib.cur_stream()))
            _lib.check(code, "moco_bn_add_relu_bwd")
        else:
            code = _timed("bn_bwd", nbytes, lambda: lib.moco_bn_add_relu_bwd2(
                dy.data_ptr(), dy2.data_ptr(), x.data_ptr(), ptr(residual), mask.data_ptr(), M, C, bn, sc,
                dx.data_ptr(), ptr(dres), ws.data_ptr(), ws.numel(), _lib.cur_stream()))
            _lib.check(code, "moco_bn_add_relu_bwd2")
        return dx, dres, dgamma, dbeta, sc_dgamma, sc_dbeta, None, None, None, None, None, None


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
        dy = _grad_rows(dy)
        dy2 = _take_handed(ctx)          # the pooled output's other consumer's gradient: summed inside the gather
        # Rebuilding the pool's input gradient inside the BatchNorm's two passes (a <= 4-window gather per element)
        # measured slower than writing it once and streaming it: the pool's backward, then the BatchNorm's.
        g = torch.empty_like(x)
        if dy2 is None:
            _lib.check(lib.moco_maxpool3x3s2_bwd(dy.data_ptr(), taps.data_ptr(), g.data_ptr(), N, H, W, C,
                                                 _lib.cur_stream()), "moco_maxpool3x3s2_bwd")
        else:
            _lib.check(lib.moco_maxpool3x3s2_bwd2(dy.data_ptr(), dy2.data_ptr(), taps.data_ptr(), g.data_ptr(), N, H, W,
                                                  C, _lib.cur_stream()), "moco_maxpool3x3s2_bwd2")
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


class _HandOverFn(torch.autograd.Function):
    """Identity in front of the second consumer of a block's input.  The input has two consumers (the first
    convolution, and the residual branch: bn3's residual or the shortcut convolution), so autograd would add their two
    bf16 gradients in a separate pass before the producer's backward reads the sum twice.  Instead the backward leaves
    this branch's gradient on the producer's node and returns None; the producer (a _BatchNormAddReluFn or the stem's
    _BatchNormReluMaxPoolFn) receives the other gradient from autograd and adds the two inside its own kernels,
    rounded to bf16 once as autograd's add would -- the sum is never written."""

    @staticmethod
    def forward(ctx, x, producer):
        ctx.producer = producer
        return x

    @staticmethod
    def backward(ctx, g):
        ctx.producer.handed = g          # this node runs before the producer's: taken by its backward (_take_handed)
        return None, None


def hand_over(x):
    """``x`` for a second consumer of ``x``; through :class:`_HandOverFn` when x's producer sums its gradients in its
    own kernels.  Anything else -- no grad, set_fused(False), a producer that is not one of those Functions -- gets x
    itself, so autograd adds the gradients as usual."""
    if not (_enabled and torch.is_grad_enabled() and x.requires_grad):
        return x
    node = x.grad_fn
    if not isinstance(node, (_BatchNormAddReluFn._backward_cls, _BatchNormReluMaxPoolFn._backward_cls)):
        return x
    return _HandOverFn.apply(x, node)


class _Conv1x1StatsFn(torch.autograd.Function):
    """y = conv2d(x, w) of a 1x1 / stride 1 convolution without bias (x bf16 channels_last, w the bf16 weight
    [Cout, Cin, 1, 1]) and the batch statistics of the training BatchNorm that reads y: one launch of
    ``moco_conv1x1_bn_stats``, which also updates that BatchNorm's running statistics.  Returns (y, mean, invstd).
    The backward is the convolution's own, ``aten.convolution_backward`` with the arguments autograd gives it for
    ``F.conv2d``, so the gradients of a given forward are unchanged.  ``producer``: x's producing node when it may
    take the input gradient together with its BatchNorm's backward reduction (:func:`_dgrad_bn_bwd`)."""

    @staticmethod
    def forward(ctx, x, w, stats, producer=None):
        lib = _lib.load()
        N, Cin, H, W = x.shape
        Cout = w.shape[0]
        y = torch.empty((N, Cout, H, W), dtype=torch.bfloat16, device=x.device, memory_format=torch.channels_last)
        mean = torch.empty(Cout, dtype=torch.float32, device=x.device)
        invstd = torch.empty_like(mean)
        ws = _workspace(x.device, conv=True)
        _lib.check(lib.moco_conv1x1_bn_stats(x.data_ptr(), w.data_ptr(), y.data_ptr(), N * H * W, Cin, Cout,
                                             _layer(None, None, mean, invstd, stats), ws.data_ptr(), ws.numel(),
                                             _lib.cur_stream()), "moco_conv1x1_bn_stats")
        ctx.save_for_backward(x, w)
        ctx.mark_non_differentiable(mean, invstd)
        ctx.producer = producer
        return y, mean, invstd

    @staticmethod
    def backward(ctx, dy, _dmean, _dinvstd):
        x, w = ctx.saved_tensors
        want_dx = ctx.needs_input_grad[0]
        g = _dgrad_bn_bwd(ctx.producer, dy, w) if ctx.producer is not None and want_dx else None
        dx, dw, _ = torch.ops.aten.convolution_backward(
            dy, x, w, None, [1, 1], [0, 0], [1, 1], False, [0, 0], 1,
            [want_dx and g is None, ctx.needs_input_grad[1], False])
        return g if g is not None else dx, dw, None, None


# (Cin, Cout) of ResNet-50's 1x1 convolutions fed by an identity block's output on which moco_conv1x1_dgrad_bn_bwd +
# the apply-only pass measured faster than cuDNN's dgrad + moco_bn_add_relu_bwd2 at batch 256: 1.37-1.43x on an H100
# SXM at a 700 W power limit (tools/conv1x1_dgrad_times.py, results/conv1x1_dgrad_times_h100.json).  These are all
# such shapes that also run their forward on moco_conv1x1_bn_stats (_CONV1X1_WINS).
_DGRAD_WINS = frozenset({(256, 64), (256, 128), (512, 128), (512, 256)})


def _dgrad_wins(M, Cin, Cout):
    """The shapes moco_conv1x1_dgrad_bn_bwd was measured to win on (_DGRAD_WINS) at batch 256's row counts."""
    return M >= 50176 and (Cin, Cout) in _DGRAD_WINS


def _dgrad_bn_bwd(node, dh, w):
    """The input gradient of a 1x1 convolution whose input is the output of ``node``, a block's residual BatchNorm
    (_BatchNormAddReluFn, identity shortcut), taken together with that BatchNorm's backward reduction: one launch of
    moco_conv1x1_dgrad_bn_bwd forms g = mask . bf16(dX + dy2) -- dy2 the gradient the hand-over left on the node --
    and the sums, and leaves (g, dgamma, dbeta) on the node for its backward (apply pass only).  None, to take
    cuDNN's dgrad, when there is no handed gradient, the block has a shortcut BN, or the shape is not in _DGRAD_WINS."""
    if getattr(node, "handed", None) is None:
        return None
    x, _, mask, weight, mean, invstd, sc_weight, _, _ = node.saved_tensors
    N, C, H, W = x.shape
    M, Cout = N * H * W, w.shape[0]
    if mask is None or sc_weight is not None or not _dgrad_wins(M, C, Cout):
        return None
    lib = _lib.load()
    dy2 = _take_handed(node)
    dh = _grad_rows(dh)
    g = torch.empty_like(x)
    dgamma = torch.empty(C, dtype=torch.float32, device=x.device)
    dbeta = torch.empty_like(dgamma)
    ws = _workspace(x.device, conv=True)
    _lib.check(lib.moco_conv1x1_dgrad_bn_bwd(
        dh.data_ptr(), w.data_ptr(), g.data_ptr(), M, C, Cout, x.data_ptr(), mask.data_ptr(), dy2.data_ptr(), None,
        _layer(weight, None, mean, invstd, dgamma=dgamma, dbeta=dbeta), None, ws.data_ptr(), ws.numel(),
        _lib.cur_stream()), "moco_conv1x1_dgrad_bn_bwd")
    node.reduced = (g, dgamma, dbeta)
    return g


# (Cin, Cout) of ResNet-50's stride-1 1x1 convolutions on which moco_conv1x1_bn_stats + the apply pass measured more
# than 3 % faster than cuDNN's convolution + the statistics and apply passes at batch 256, on an H100 SXM at a 700 W
# power limit (tools/conv1x1_times.py, results/conv1x1_times_h100.json): 1.08-1.23x on stages 1-2 and on the 256 -> 1024
# conv3 of stage 3.  The K-heavy ones of stages 3-4 (1024 -> 256, 1024 -> 512, 2048 -> 512, 512 -> 2048) measured
# 0.73-0.97x and keep cuDNN.
_CONV1X1_WINS = frozenset({(64, 64), (256, 64), (64, 256), (256, 128), (512, 128), (128, 512), (512, 256),
                           (256, 1024)})


def _conv1x1_wins(M, Cin, Cout):
    """The shapes moco_conv1x1_bn_stats was measured to win on (_CONV1X1_WINS) at batch 256's row counts; smaller
    batches were not measured and keep cuDNN."""
    return M >= 50176 and (Cin, Cout) in _CONV1X1_WINS


def _conv1x1_ok(conv, bn, x, residual=None, shortcut_bn=None):
    """conv(x) may run as moco_conv1x1_bn_stats: a 1x1 / stride 1 convolution without bias, groups, dilation or
    padding computing in bf16 on bf16 channels_last activations, channels multiples of 64, and bn (with ``residual``,
    and ``shortcut_bn`` on ``residual`` when bn is a downsample block's bn3) taking its training kernels on the
    output."""
    w = conv.weight
    if not (_enabled and isinstance(conv, nn.Conv2d) and type(conv).forward is nn.Conv2d.forward
            and conv.kernel_size == (1, 1) and conv.stride == (1, 1) and conv.padding == (0, 0)
            and conv.dilation == (1, 1) and conv.groups == 1 and conv.bias is None and _rows_ok(x)
            and w.is_cuda and w.device == x.device and x.shape[1] == w.shape[1]):
        return False
    if not (w.dtype == torch.bfloat16 or (torch.is_autocast_enabled("cuda")
                                         and torch.get_autocast_dtype("cuda") == torch.bfloat16)):
        return False
    N, Cin, H, W = x.shape
    Cout = w.shape[0]
    out = torch.Size((N, Cout, H, W))
    if Cin % 64 != 0 or Cout % 64 != 0 or not bn._fusable_shape(out, residual):
        return False
    if shortcut_bn is not None and not (bn.relu and not shortcut_bn.relu and shortcut_bn._fusable(residual, None)):
        return False
    return _conv1x1_wins(N * H * W, Cin, Cout)


def conv1x1_stats(conv, bn, x, residual=None, shortcut_bn=None, handed_over=False):
    """(conv(x), stats): stats = the batch statistics of the training BatchNorm ``bn`` on conv(x), computed with the
    convolution by moco_conv1x1_bn_stats (``bn``'s running statistics are updated), to be passed to ``bn(...,
    stats=stats)``; None where that kernel does not take the convolution (see :func:`_conv1x1_ok`), which then runs
    as ``conv(x)``.  ``residual`` / ``shortcut_bn``: what ``bn`` will be called with.  ``handed_over``: x's only
    other consumer is ``hand_over(x)``; when x is a block's residual BatchNorm output, the backward may then take the
    input gradient with that BatchNorm's reduction (:func:`_dgrad_bn_bwd`)."""
    if not _conv1x1_ok(conv, bn, x, residual, shortcut_bn):
        return conv(x), None
    w = conv.weight.to(torch.bfloat16).contiguous()     # outside the Function: its autograd gives the fp32 gradient
    node = x.grad_fn if handed_over else None
    producer = node if isinstance(node, _BatchNormAddReluFn._backward_cls) else None
    y, mean, invstd = _Conv1x1StatsFn.apply(x, w, bn._stats(), producer)
    return y, (mean, invstd)


# (Cin, Cout, key, shortcut) of ResNet-50's conv3 -> bn3 on which moco_conv1x1_bn_add_relu_fwd measured more than 3 %
# faster than moco_conv1x1_bn_stats + moco_bn_fwd_train_given at batch 256, on an H100 SXM at a 700 W power limit
# (tools/conv1x1_apply_times.py, results/conv1x1_apply_times_h100.json): 1.06-1.37x.  key: the forward without a
# backward (the key encoder), where conv3's output is never written; otherwise the query encoder's, where the
# statistics pass still writes it for bn3's backward.  shortcut: a downsample block (the shortcut BN in the apply).
# Stage 3's downsample block in the query encoder measured 0.98x and keeps the apply pass.
_APPLY_WINS = frozenset({(64, 256, False, False), (128, 512, False, False), (256, 1024, False, False),
                         (64, 256, False, True), (128, 512, False, True),
                         (64, 256, True, False), (128, 512, True, False), (256, 1024, True, False),
                         (64, 256, True, True), (128, 512, True, True), (256, 1024, True, True)})


def _apply_wins(M, Cin, Cout, key, shortcut):
    return M >= 50176 and (Cin, Cout, key, shortcut) in _APPLY_WINS


def conv1x1_bn_add_relu(conv, bn, x, residual, shortcut_bn=None, sc_stats=None, avgpool=False):
    """``bn(conv(x), residual, shortcut_bn=shortcut_bn, avgpool=avgpool, ...)``: a bottleneck's conv3 -> bn3, with
    ``sc_stats`` the shortcut BN's statistics from :func:`conv1x1_stats` (None where it did not take the shortcut).
    Where :func:`conv1x1_stats` takes conv and the shape is in _APPLY_WINS, bn3 is applied by
    moco_conv1x1_bn_add_relu_fwd, which recomputes conv(x) rather than reading it back.  With a backward to follow
    (the query encoder) conv1x1_stats still writes conv(x), which bn3's backward reads; without one (the key encoder)
    the statistics pass runs inside the same call without a store, and conv(x) is never allocated.  Same values,
    running statistics and launch count as the path it replaces."""
    if not avgpool and bn.relu and residual is not None and _conv1x1_ok(conv, bn, x, residual, shortcut_bn):
        params = (x, residual, conv.weight, bn.weight, bn.bias) + (
            (shortcut_bn.weight, shortcut_bn.bias) if shortcut_bn is not None else ())
        key = not (torch.is_grad_enabled() and any(t.requires_grad for t in params))
        N, Cin, H, W = x.shape
        if _apply_wins(N * H * W, Cin, conv.weight.shape[0], key, shortcut_bn is not None):
            w = conv.weight.to(torch.bfloat16).contiguous()
            if key:
                return _conv_bn_add_relu_nograd(x, w, bn, residual, shortcut_bn, sc_stats)
            h, mean, invstd = _Conv1x1StatsFn.apply(x, w, bn._stats(), None)
            return bn._add_relu(h, residual, shortcut_bn, (mean, invstd), sc_stats, recompute=(x, w))
    h, st = conv1x1_stats(conv, bn, x, residual, shortcut_bn)
    return bn(h, residual, shortcut_bn=shortcut_bn, avgpool=avgpool, stats=st, sc_stats=sc_stats)


def _conv_bn_add_relu_nograd(x, w, bn, residual, shortcut_bn, sc_stats):
    """relu(bn(conv2d(x, w)) + r) for a forward without a backward: one moco_conv1x1_bn_add_relu_fwd call runs the
    statistics pass (no store) and the recomputing apply pass, plus the shortcut BN's statistics unless given."""
    lib = _lib.load()
    N, Cin, H, W = x.shape
    C, M = w.shape[0], N * H * W
    y = torch.empty((N, C, H, W), dtype=torch.bfloat16, device=x.device, memory_format=torch.channels_last)
    f32 = lambda: torch.empty(C, dtype=torch.float32, device=x.device)
    mean, invstd = f32(), f32()                     # kept alive until the call: the layer holds raw pointers
    layer = _layer(bn.weight, bn.bias, mean, invstd, bn._stats())
    sc, flags = None, 0
    if shortcut_bn is not None:
        sc_mean, sc_invstd = sc_stats if sc_stats is not None else (f32(), f32())
        sc = _layer(shortcut_bn.weight, shortcut_bn.bias, sc_mean, sc_invstd, shortcut_bn._stats())
        flags = _lib.BN_SC_STATS_GIVEN if sc_stats is not None else 0
    ws = _workspace(x.device)
    # algorithmic bytes: both passes read x; the apply reads the residual (+ the shortcut input for its statistics)
    # and writes y
    nbytes = M * 2 * (2 * Cin + C * (2 + (sc is not None and sc_stats is None)))
    code = _timed("bn_fwd", nbytes, lambda: lib.moco_conv1x1_bn_add_relu_fwd(
        x.data_ptr(), w.data_ptr(), residual.data_ptr(), y.data_ptr(), None, M, Cin, C, layer, sc, flags,
        ws.data_ptr(), ws.numel(), _lib.cur_stream()))
    _lib.check(code, "moco_conv1x1_bn_add_relu_fwd")
    return y


class BatchNormAct2d(nn.BatchNorm2d):
    """``nn.BatchNorm2d`` + optional residual add + optional ReLU (``forward(x, residual=None)``)."""

    def __init__(self, num_features, relu=False, **kw):
        super().__init__(num_features, **kw)
        self.relu = bool(relu)
        self.frozen = False             # MoCoResNet.freeze(): eval mode without grad runs the eval kernels
        self._fold_key = None
        self._fold = None

    def _fusable(self, x, residual):
        return _rows_ok(x) and self._fusable_shape(x.shape, residual)

    def _fusable_shape(self, shape, residual):
        """The training kernels take a bf16 channels_last input of this shape (and this residual)."""
        C = self.num_features
        return (_enabled and self.training and self.affine and self.momentum is not None
                and (residual is None or (_rows_ok(residual) and residual.shape == shape))
                and 64 <= C <= 2048 and (C & (C - 1)) == 0 and shape[1] == C
                and shape.numel() // C > 1             # a single value per channel: nn.BatchNorm2d's own error
                and self.weight.dtype == torch.float32 and self.weight.is_cuda
                and (self.running_mean is None or self.running_mean.dtype == torch.float32))

    def _eval_ok(self, x, residual):
        """The frozen path: eval mode, grad mode off, running statistics, and activations the kernels take."""
        C = self.num_features
        return (_enabled and self.frozen and not self.training and not torch.is_grad_enabled() and self.affine
                and self.track_running_stats and self.running_mean is not None
                and _rows_ok(x) and (residual is None or _rows_ok(residual, x))
                and 64 <= C <= 2048 and (C & (C - 1)) == 0 and x.shape[1] == C
                and self.weight.dtype == torch.float32 and self.weight.is_cuda
                and self.running_var.dtype == torch.float32)

    def folded(self):
        """(scale, shift) fp32 [C]: weight / sqrt(running_var + eps) and bias - running_mean * scale.  Cached, and
        re-folded whenever the weight, the bias or a running buffer is replaced or modified in place through the
        tensor itself (``load_state_dict``, ``copy_``, optimizer steps): the cache key is each tensor's storage and
        version counter.  Writes through ``.data`` do not advance the version counter; call
        ``MoCoResNet.freeze()`` again after them, which drops the cached coefficients."""
        ts = (self.weight, self.bias, self.running_mean, self.running_var)
        key = tuple((t.data_ptr(), t._version) for t in ts) + (self.eps,)
        if key != self._fold_key:
            with torch.no_grad():
                scale = self.weight.float() / torch.sqrt(self.running_var.float() + self.eps)
                shift = self.bias.float() - self.running_mean.float() * scale
            self._fold, self._fold_key = (scale.contiguous(), shift.contiguous()), key
        return self._fold

    def _eval(self, x, residual, sc, avgpool):
        lib = _lib.load()
        N, C, H, W = x.shape
        scale, shift = self.folded()
        sc_scale, sc_shift = sc.folded() if sc is not None else (None, None)
        ptr = lambda t: t.data_ptr() if t is not None else None
        # algorithmic bytes: reads x (+ residual), writes y (or the pooled fp32 features)
        reads = N * H * W * C * 2 * (1 + (residual is not None))
        if avgpool:
            y = torch.empty((N, C), dtype=torch.float32, device=x.device)
            code = _timed("bn_eval", reads + N * C * 4, lambda: lib.moco_bn_eval_act_avgpool(
                x.data_ptr(), ptr(residual), y.data_ptr(), N, H * W, C, scale.data_ptr(), shift.data_ptr(),
                int(self.relu), ptr(sc_scale), ptr(sc_shift), _lib.cur_stream()))
            _lib.check(code, "moco_bn_eval_act_avgpool")
            return y
        y = torch.empty_like(x)
        code = _timed("bn_eval", reads + N * H * W * C * 2, lambda: lib.moco_bn_eval_act(
            x.data_ptr(), ptr(residual), y.data_ptr(), N * H * W, C, scale.data_ptr(), shift.data_ptr(),
            int(self.relu), ptr(sc_scale), ptr(sc_shift), _lib.cur_stream()))
        _lib.check(code, "moco_bn_eval_act")
        return y

    def _stats(self):
        return (self.running_mean, self.running_var, self.num_batches_tracked if self.track_running_stats else None,
                self.momentum, self.eps)

    def forward(self, x, residual=None, shortcut_bn=None, avgpool=False, stats=None, sc_stats=None):
        """``shortcut_bn``: a downsample block's shortcut BatchNorm (no ReLU); ``residual`` is then its input, the
        shortcut convolution's raw output, and ``y = relu?(bn(x) + shortcut_bn(residual))``.  ``avgpool``: return
        the global average pool of y, flattened to [N, C] (fp32 from the frozen path, y's dtype otherwise).
        ``stats`` / ``sc_stats``: the batch statistics of x / of the shortcut input from :func:`conv1x1_stats`, which
        only gives them where the training kernels take this call."""
        if avgpool:
            if (shortcut_bn is None or not shortcut_bn.relu and shortcut_bn._eval_ok(residual, None)) \
                    and self._eval_ok(x, residual) and stats is None and sc_stats is None:
                return self._eval(x, residual, shortcut_bn, True)
            return torch.flatten(F.adaptive_avg_pool2d(self.forward(x, residual, shortcut_bn, stats=stats,
                                                                    sc_stats=sc_stats), 1), 1)
        if shortcut_bn is not None:
            if (not shortcut_bn.relu and self._eval_ok(x, residual) and shortcut_bn._eval_ok(residual, None)
                    and stats is None and sc_stats is None):
                return self._eval(x, residual, shortcut_bn, False)
            if (self.relu and not shortcut_bn.relu and self._fusable(x, residual)
                    and shortcut_bn._fusable(residual, None)):
                return self._add_relu(x, residual, shortcut_bn, stats, sc_stats)
            residual = shortcut_bn(residual, stats=sc_stats)
        if self._eval_ok(x, residual) and stats is None:
            return self._eval(x, residual, None, False)
        if self._fusable(x, residual):
            if self.relu and residual is not None:
                return self._add_relu(x, residual, None, stats)
            return _BatchNormActFn.apply(x, self.weight, self.bias, residual, self.running_mean, self.running_var,
                                         self.num_batches_tracked if self.track_running_stats else None,
                                         self.momentum, self.eps, self.relu, stats)
        if stats is not None:
            raise RuntimeError("moco_b200: batch statistics given to a BatchNorm that cannot take them")
        y = super().forward(x)
        if residual is not None:
            y = y + residual
        return F.relu(y, inplace=True) if self.relu else y

    def forward_maxpool(self, x, pool):
        """``pool(self(x))`` for a :class:`MaxPool3x3s2` ``pool`` (the stem): one pass applies the BatchNorm + ReLU to
        every tap of the pool, so that the BatchNorm's output is never written."""
        if self.relu and isinstance(pool, MaxPool3x3s2) and self._eval_ok(x, None):
            lib = _lib.load()
            N, C, H, W = x.shape
            OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
            y = torch.empty((N, C, OH, OW), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
            scale, shift = self.folded()
            # algorithmic bytes: the pool pass reads x and writes y
            code = _timed("bn_eval", N * H * W * C * 2 + N * OH * OW * C * 2, lambda: lib.moco_bn_relu_maxpool_eval(
                x.data_ptr(), y.data_ptr(), N, H, W, C, scale.data_ptr(), shift.data_ptr(), _lib.cur_stream()))
            _lib.check(code, "moco_bn_relu_maxpool_eval")
            return y
        if self.relu and isinstance(pool, MaxPool3x3s2) and self._fusable(x, None):
            return _BatchNormReluMaxPoolFn.apply(x, self.weight, self.bias, self._stats())
        return pool(self(x))

    def _add_relu(self, x, residual, sc, stats=None, sc_stats=None, recompute=None):
        params = (x, residual, self.weight, self.bias) + ((sc.weight, sc.bias) if sc is not None else ())
        want_mask = torch.is_grad_enabled() and any(t.requires_grad for t in params)
        return _BatchNormAddReluFn.apply(x, residual, self.weight, self.bias,
                                         sc.weight if sc is not None else None, sc.bias if sc is not None else None,
                                         self._stats(), sc._stats() if sc is not None else None, want_mask,
                                         stats, sc_stats, recompute)

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
