"""BatchNorm2d with the block's ReLU / residual add folded in, on this library's channels_last bf16 kernels.

The reference's encoders apply ``nn.BatchNorm2d`` -> [``out += residual``] -> [``nn.ReLU``] at
``moco/models/resnet.py:42-63,74-102,114,139-143,156-157``; ShuffleBN (``moco/util.py:69-93``) exists for exactly these
batch statistics, and left to ATen's channels_last kernels they take most of the GPU time of a step.  :class:`BatchNormAct2d` is an ``nn.BatchNorm2d`` (same parameters,
buffers and ``state_dict`` keys, same running-statistics updates) whose training-mode forward / backward on CUDA
bf16 channels_last activations are two launches each of ``csrc/bn_nhwc.cu``: ``moco_bn_fwd_train_given``
(:func:`_bn_fwd`) and ``moco_bn_bwd`` (:func:`_bn_bwd`).
A block's residual BatchNorm, ``relu(bn(x) + r)``, has the forward write the ReLU mask as bits and the backward read
them (``moco_bn_add_relu_bwd``) rather than re-read ``y``, and in a downsample block (``forward(x, residual,
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


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _f32(C, device):
    return torch.empty(C, dtype=torch.float32, device=device)


def _layer(weight, bias, mean, invstd, stats=None, dgamma=None, dbeta=None):
    """moco_bn_layer of one BatchNorm: stats = (running_mean, running_var, num_batches_tracked, momentum, eps)."""
    rm, rv, nbt, momentum, eps = stats if stats is not None else (None, None, None, 0.0, 0.0)
    return _lib.BnLayer(_ptr(weight), _ptr(bias), _ptr(rm), _ptr(rv), _ptr(nbt), float(momentum), float(eps),
                        _ptr(mean), _ptr(invstd), _ptr(dgamma), _ptr(dbeta))


def _bn_fwd(x, residual, y, mask, relu, bn, sc=None, given=None, sc_given=None, recompute=None):
    """The training forward into ``y`` (and the ReLU mask bits into ``mask``): y = relu?(bn(x) [+ r]), r = residual
    or, with ``sc``, bf16(sc(residual)).  bn / sc: (weight, bias, stats as for :func:`_layer`).  given / sc_given:
    (mean, invstd) the producing convolution computed (:func:`conv1x1_stats`, which also updated the running
    statistics); that layer's statistics pass is skipped.  recompute: (a, w) with x = conv2d(a, w) of a 1x1
    convolution: moco_conv1x1_bn_add_relu_fwd computes y from a instead of reading x, which may then be None when
    its statistics are not given either.  Returns (mean, invstd, sc_mean, sc_invstd)."""
    lib = _lib.load()
    N, C, H, W = y.shape
    M = N * H * W
    mean, invstd = given if given is not None else (_f32(C, y.device), _f32(C, y.device))
    layer = _layer(bn[0], bn[1], mean, invstd, bn[2])
    sc_layer, sc_mean, sc_invstd = None, None, None
    if sc is not None:
        sc_mean, sc_invstd = sc_given if sc_given is not None else (_f32(C, y.device), _f32(C, y.device))
        sc_layer = _layer(sc[0], sc[1], sc_mean, sc_invstd, sc[2])
    flags = (_lib.BN_STATS_GIVEN if given is not None else 0) | (_lib.BN_SC_STATS_GIVEN if sc_given is not None else 0)
    ws = _workspace(y.device)
    # algorithmic bytes: a statistics pass reads its layer's input; the apply pass reads x (+ residual) and writes y
    # (+ mask bits).  recompute: both of bn's passes read a in place of x.
    sc_pass = sc is not None and sc_given is None
    mask_bytes = M * C // 8 if mask is not None else 0
    if recompute is not None:
        a, w = recompute
        Cin = a.shape[1]
        name = "moco_conv1x1_bn_add_relu_fwd"
        nbytes = 2 * M * (Cin * (1 + (given is None)) + C * (2 + sc_pass)) + mask_bytes
        args = (a.data_ptr(), w.data_ptr(), residual.data_ptr(), y.data_ptr(), _ptr(mask), M, Cin, C, layer, sc_layer,
                flags, ws.data_ptr(), ws.numel())
    else:
        name = "moco_bn_fwd_train_given"
        nbytes = 2 * M * C * (2 + (residual is not None) + (given is None) + sc_pass) + mask_bytes
        args = (x.data_ptr(), _ptr(residual), y.data_ptr(), _ptr(mask), M, C, int(relu), layer, sc_layer, flags,
                ws.data_ptr(), ws.numel())
    _lib.check(_timed("bn_fwd", nbytes, lambda: getattr(lib, name)(*args, _lib.cur_stream())), name)
    return mean, invstd, sc_mean, sc_invstd


def _bn_bwd(dy, x, bn, relu, has_res=False, y=None, mask=None, dy2=None, sc=None, dres=None, sums=None):
    """The training backward of :func:`_bn_fwd`.  bn: (weight, bias, mean, invstd); sc: (weight, mean, invstd, input)
    of the shortcut BN.  The ReLU mask is ``mask``, the forward's bits, else taken from ``y`` (relu and has_res) or
    recomputed from x (relu).  dy2: a second gradient of y, summed with dy inside both passes.  dres: where the
    masked gradient -- with sc, the shortcut BN's input gradient -- is written.  sums: (dgamma, dbeta) of an
    already masked dy (:func:`_dgrad_bn_bwd`): the element-wise pass alone.
    Returns (dx, dgamma, dbeta, sc_dgamma, sc_dbeta)."""
    lib = _lib.load()
    N, C, H, W = x.shape
    M = N * H * W
    weight, bias, mean, invstd = bn
    dx = torch.empty_like(x)
    dgamma, dbeta = sums if sums is not None else (_f32(C, x.device), _f32(C, x.device))
    layer = _layer(weight, bias, mean, invstd, dgamma=dgamma, dbeta=dbeta)
    sc_layer, sc_dgamma, sc_dbeta, x2 = None, None, None, None
    if sc is not None:
        sc_weight, sc_mean, sc_invstd, x2 = sc
        sc_dgamma, sc_dbeta = _f32(C, x.device), _f32(C, x.device)
        sc_layer = _layer(sc_weight, None, sc_mean, sc_invstd, dgamma=sc_dgamma, dbeta=sc_dbeta)
    ws = _workspace(x.device)
    # algorithmic bytes: the reduce and the apply pass each read dy (+ dy2), x (+ y | mask bits) (+ the shortcut
    # input); the apply pass writes dx (+ d residual)
    passes = 1 if sums is not None else 2
    reads = 2 + (y is not None) + (x2 is not None) + (dy2 is not None)
    nbytes = 2 * M * C * (passes * reads + 1 + (dres is not None)) + (2 * (M * C // 8) if mask is not None else 0)
    tail = (ws.data_ptr(), ws.numel())
    if sums is not None:
        name = "moco_bn_bwd_apply_given"
        args = (dy.data_ptr(), x.data_ptr(), None, M, C, layer, None, dx.data_ptr(), None)
    elif mask is None:
        name = "moco_bn_bwd"
        args = (dy.data_ptr(), x.data_ptr(), _ptr(y), M, C, weight.data_ptr(), bias.data_ptr(), mean.data_ptr(),
                invstd.data_ptr(), int(relu), int(has_res), dx.data_ptr(), _ptr(dres), dgamma.data_ptr(),
                dbeta.data_ptr()) + tail
    else:
        name = "moco_bn_add_relu_bwd" if dy2 is None else "moco_bn_add_relu_bwd2"
        grads = (dy.data_ptr(),) if dy2 is None else (dy.data_ptr(), dy2.data_ptr())
        args = grads + (x.data_ptr(), _ptr(x2), mask.data_ptr(), M, C, layer, sc_layer, dx.data_ptr(),
                        _ptr(dres)) + tail
    _lib.check(_timed("bn_bwd", nbytes, lambda: getattr(lib, name)(*args, _lib.cur_stream())), name)
    return dx, dgamma, dbeta, sc_dgamma, sc_dbeta


class _BatchNormActFn(torch.autograd.Function):
    """y = relu?(batch_norm_train(x) [+ residual]); x, residual, y bf16 channels_last; weight / bias fp32."""

    @staticmethod
    def forward(ctx, x, weight, bias, residual, running_mean, running_var, num_batches_tracked, momentum, eps, relu,
                given=None):
        """given: (mean, invstd) already computed by the producing convolution (:func:`conv1x1_stats`), which also
        updated the running statistics: only the apply pass runs."""
        y = torch.empty_like(x)                                   # keeps the channels_last strides
        stats = (running_mean, running_var, num_batches_tracked, momentum, eps)
        mean, invstd, _, _ = _bn_fwd(x, residual, y, None, relu, (weight, bias, stats), given=given)
        ctx.relu = bool(relu)
        ctx.has_res = residual is not None
        # the ReLU mask of the backward is recomputed from x unless a residual went into it
        ctx.save_for_backward(x, y if (relu and residual is not None) else None, weight, bias, mean, invstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y, weight, bias, mean, invstd = ctx.saved_tensors
        dy = _grad_rows(dy)
        want_res = ctx.has_res and ctx.needs_input_grad[3]
        dres = torch.empty_like(x) if want_res and ctx.relu else None
        dx, dgamma, dbeta, _, _ = _bn_bwd(dy, x, (weight, bias, mean, invstd), ctx.relu, ctx.has_res, y=y, dres=dres)
        if want_res and not ctx.relu:
            dres = dy                                             # without a ReLU the residual's gradient is dy itself
        return dx, dgamma, dbeta, dres, None, None, None, None, None, None, None


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
        N, C, H, W = x.shape
        y = torch.empty_like(x)
        mask = torch.empty((N * H * W, C // 8), dtype=torch.uint8, device=x.device) if want_mask else None
        sc = (sc_weight, sc_bias, sc_stats) if sc_weight is not None else None
        mean, invstd, sc_mean, sc_invstd = _bn_fwd(x, residual, y, mask, True, (weight, bias, stats), sc, given,
                                                   sc_given, recompute)
        ctx.save_for_backward(x, residual if sc is not None else None, mask, weight, mean, invstd, sc_weight, sc_mean,
                              sc_invstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, residual, mask, weight, mean, invstd, sc_weight, sc_mean, sc_invstd = ctx.saved_tensors
        if mask is None:
            raise RuntimeError("moco_b200: BatchNormAct2d ran its forward without the ReLU mask (no input required grad)")
        dy = _grad_rows(dy)
        bn = (weight, None, mean, invstd)
        reduced, ctx.reduced = getattr(ctx, "reduced", None), None
        if reduced is not None and dy.data_ptr() == reduced[0].data_ptr():
            # the consumer's dgrad formed g = dy and the sums (_dgrad_bn_bwd); another consumer adding to the gradient
            # gives a different tensor, which takes the full backward below (g is already masked: mask(g + e) = g +
            # mask(e))
            g, dgamma, dbeta = reduced
            dx = _bn_bwd(g, x, bn, False, sums=(dgamma, dbeta))[0]
            return (dx, g if ctx.needs_input_grad[1] else None, dgamma, dbeta, None, None, None, None, None, None, None,
                    None)
        dy2 = _take_handed(ctx)          # y's other consumer's gradient: summed inside both passes
        sc = (sc_weight, sc_mean, sc_invstd, residual) if sc_weight is not None else None
        dres = torch.empty_like(x) if sc is not None or ctx.needs_input_grad[1] else None
        dx, dgamma, dbeta, sc_dgamma, sc_dbeta = _bn_bwd(dy, x, bn, True, mask=mask, dy2=dy2, sc=sc, dres=dres)
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
        mean, invstd = _f32(C, x.device), _f32(C, x.device)
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
        dx, dgamma, dbeta, _, _ = _bn_bwd(g, x, (weight, bias, mean, invstd), True)
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
        mean, invstd = _f32(Cout, x.device), _f32(Cout, x.device)
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
# the fewest rows N * H * W of a shape in the _*_WINS tables at the batch they were measured at: 256 x 14 x 14
_BATCH256_ROWS = 50176


def _dgrad_wins(M, Cin, Cout):
    """The shapes moco_conv1x1_dgrad_bn_bwd was measured to win on (_DGRAD_WINS) at batch 256's row counts."""
    return M >= _BATCH256_ROWS and (Cin, Cout) in _DGRAD_WINS


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
    dgamma, dbeta = _f32(C, x.device), _f32(C, x.device)
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
    return M >= _BATCH256_ROWS and (Cin, Cout) in _CONV1X1_WINS


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
    return M >= _BATCH256_ROWS and (Cin, Cout, key, shortcut) in _APPLY_WINS


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
    N, Cin, H, W = x.shape
    y = torch.empty((N, w.shape[0], H, W), dtype=torch.bfloat16, device=x.device, memory_format=torch.channels_last)
    sc = (shortcut_bn.weight, shortcut_bn.bias, shortcut_bn._stats()) if shortcut_bn is not None else None
    _bn_fwd(None, residual, y, None, True, (bn.weight, bn.bias, bn._stats()), sc, None, sc_stats, recompute=(x, w))
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

    def _envelope_ok(self, shape):
        """What the training and the frozen kernels both need of the module and of the input's channels."""
        C = self.num_features
        return (_enabled and self.affine and 64 <= C <= 2048 and (C & (C - 1)) == 0 and shape[1] == C
                and self.weight.dtype == torch.float32 and self.weight.is_cuda)

    def _fusable_shape(self, shape, residual):
        """The training kernels take a bf16 channels_last input of this shape (and this residual)."""
        return (self._envelope_ok(shape) and self.training and self.momentum is not None
                and (residual is None or (_rows_ok(residual) and residual.shape == shape))
                and shape.numel() // self.num_features > 1    # a single value per channel: nn.BatchNorm2d's own error
                and (self.running_mean is None or self.running_mean.dtype == torch.float32))

    def _eval_ok(self, x, residual):
        """The frozen path: eval mode, grad mode off, running statistics, and activations the kernels take."""
        return (self.frozen and not self.training and not torch.is_grad_enabled()
                and self.track_running_stats and self.running_mean is not None
                and _rows_ok(x) and (residual is None or _rows_ok(residual, x)) and self._envelope_ok(x.shape)
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
        # algorithmic bytes: reads x (+ residual), writes y (or the pooled fp32 features)
        reads = N * H * W * C * 2 * (1 + (residual is not None))
        if avgpool:
            y = torch.empty((N, C), dtype=torch.float32, device=x.device)
            code = _timed("bn_eval", reads + N * C * 4, lambda: lib.moco_bn_eval_act_avgpool(
                x.data_ptr(), _ptr(residual), y.data_ptr(), N, H * W, C, scale.data_ptr(), shift.data_ptr(),
                int(self.relu), _ptr(sc_scale), _ptr(sc_shift), _lib.cur_stream()))
            _lib.check(code, "moco_bn_eval_act_avgpool")
            return y
        y = torch.empty_like(x)
        code = _timed("bn_eval", reads + N * H * W * C * 2, lambda: lib.moco_bn_eval_act(
            x.data_ptr(), _ptr(residual), y.data_ptr(), N * H * W, C, scale.data_ptr(), shift.data_ptr(),
            int(self.relu), _ptr(sc_scale), _ptr(sc_shift), _lib.cur_stream()))
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
        dy = _grad_rows(dy)
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
