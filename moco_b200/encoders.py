"""Query / key encoders for the MoCo step (host PyTorch, as BASELINE.json:north_star keeps them).

Plain ResNet-18/34/50 with the MoCo head of the reference's variant
(``moco/models/resnet.py:109,125-126,177-178``: ``fc`` to ``low_dim`` followed by
L2 normalisation).  Out of the hot-path scope (SURVEY §2 row 5) -- these exist to
drive the end-to-end step / benchmark; the convolutions are cuDNN via PyTorch.  The
BatchNorm -> (+ residual) -> ReLU groups (resnet.py:42-63,74-102,156-157) are
:class:`moco_b200.bn.BatchNormAct2d`: an ``nn.BatchNorm2d`` (same parameters / buffers /
state_dict keys) that runs this library's fused channels_last bf16 kernels in training
mode on CUDA and ``nn.BatchNorm2d``'s own forward everywhere else; the stem's max pooling
(resnet.py:119) is :class:`moco_b200.bn.MaxPool3x3s2` on the same terms.
"""
from __future__ import annotations

import torch
from torch import nn
import torch.nn.functional as F

from . import bn as bn_mod
from .bn import BatchNormAct2d, MaxPool3x3s2
from .util import crop_to_s2d_bf16


class _Basic(nn.Module):
    expansion = 1

    def __init__(self, cin, planes, stride):
        super().__init__()
        self.conv1 = nn.Conv2d(cin, planes, 3, stride, 1, bias=False)
        self.bn1 = BatchNormAct2d(planes, relu=True)
        self.conv2 = nn.Conv2d(planes, planes, 3, 1, 1, bias=False)
        self.bn2 = BatchNormAct2d(planes, relu=True)              # relu(bn(.) + residual)
        self.short = None
        if stride != 1 or cin != planes:
            self.short = nn.Sequential(nn.Conv2d(cin, planes, 1, stride, bias=False), BatchNormAct2d(planes))

    def forward(self, x, avgpool=False):
        y = self.bn1(self.conv1(x))
        r = bn_mod.hand_over(x)                   # x's second consumer: its gradient is summed in x's producer
        if self.short is None:
            return self.bn2(self.conv2(y), r, avgpool=avgpool)
        return self.bn2(self.conv2(y), self.short[0](r), shortcut_bn=self.short[1], avgpool=avgpool)   # one BN group


class _Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, cin, planes, stride):
        super().__init__()
        cout = planes * 4
        self.conv1 = nn.Conv2d(cin, planes, 1, bias=False)
        self.bn1 = BatchNormAct2d(planes, relu=True)
        self.conv2 = nn.Conv2d(planes, planes, 3, stride, 1, bias=False)
        self.bn2 = BatchNormAct2d(planes, relu=True)
        self.conv3 = nn.Conv2d(planes, cout, 1, bias=False)
        self.bn3 = BatchNormAct2d(cout, relu=True)                # relu(bn(.) + residual)
        self.short = None
        if stride != 1 or cin != cout:
            self.short = nn.Sequential(nn.Conv2d(cin, cout, 1, stride, bias=False), BatchNormAct2d(cout))

    def forward(self, x, avgpool=False):
        """``avgpool``: return the global average pool of the output, [N, C] (the last block of the trunk).  The 1x1
        convolutions take the following BatchNorm's batch statistics with them where they can (bn.conv1x1_stats)."""
        h, st = bn_mod.conv1x1_stats(self.conv1, self.bn1, x, handed_over=True)   # x's other consumer: hand_over
        y = self.bn1(h, stats=st)
        y = self.bn2(self.conv2(y))
        r = bn_mod.hand_over(x)                   # x's second consumer: its gradient is summed in x's producer
        if self.short is None:
            return bn_mod.conv1x1_bn_add_relu(self.conv3, self.bn3, y, r, avgpool=avgpool)
        s, sc_st = bn_mod.conv1x1_stats(self.short[0], self.short[1], r)
        return bn_mod.conv1x1_bn_add_relu(self.conv3, self.bn3, y, s, self.short[1], sc_st, avgpool)   # one BN group


class StemConv(nn.Conv2d):
    """The reference's first convolution (moco/models/resnet.py:112: 3 -> 64, 7x7, stride 2, padding 3, no bias) with
    the same weight parameter.  Given the usual [N, 3, H, W] input it is that convolution.  Given the 16-channel
    space-to-depth input that ``moco_crop_s2d_bf16`` writes ([N, 16, H/2+3, W/2+3], see include/moco_b200.h) it runs
    the EQUIVALENT 4x4 / stride 1 convolution with the weights re-indexed on the fly,
        w'[o, (b*2+d)*3 + c, a, e] = w[o, c, 2a+b-1, 2e+d-1]        (taps -1 are zero),
    which is differentiable w.r.t. the 7x7 parameter -- so cuDNN sees 16 input channels (its implicit-GEMM
    kernels) instead of 3 (a legacy kernel at 2 % of peak + channel-padding passes)."""

    def __init__(self):
        super().__init__(3, 64, 7, 2, 3, bias=False)

    def s2d_weight(self):
        w8 = F.pad(self.weight, (1, 0, 1, 0)).view(64, 3, 4, 2, 4, 2)          # [o, c, a, b, e, d]
        return F.pad(w8.permute(0, 3, 5, 1, 2, 4).reshape(64, 12, 4, 4), (0, 0, 0, 0, 0, 4))

    def forward(self, x):
        if x.shape[1] == 16:
            return F.conv2d(x, self.s2d_weight(), None, 1, 0)
        return super().forward(x)


class MoCoResNet(nn.Module):
    """ResNet trunk -> global average pool -> fc(low_dim) -> L2 normalise.

    ``forward(x, layer)`` exits early as the reference's ``ResNet.forward(x, layer)`` (resnet.py:152-180) does, which
    its linear evaluation uses: layer <= 0 the input, 1 the stem's max-pool output, 2..5 the output of stage 1..4, 6
    the pooled and flattened features, 7 (default) the fc output, L2-normalised unless ``l2norm`` is off.
    ``freeze()`` prepares the model for that evaluation (see its docstring).

    ``mlp=True`` gives MoCo v2's projection head: ``fc`` is Linear(C, C) -> ReLU -> Linear(C, low_dim), state-dict
    keys ``fc.0.*`` and ``fc.2.*`` as in MoCo v2's checkpoints; the default is the bare Linear.  ``feat_dim`` (C) and
    ``low_dim`` are the widths of layers 6 and 7 either way."""

    def __init__(self, block, depths, low_dim=128, width=1, mlp=False):
        super().__init__()
        base = int(64 * width)
        # index 2 was the separate ReLU; kept as a placeholder so that the state_dict keys do not move
        self.stem = nn.Sequential(StemConv(), BatchNormAct2d(64, relu=True), nn.Identity(),
                                  MaxPool3x3s2())
        layers, cin = [], 64
        for i, d in enumerate(depths):
            planes = base * (2 ** i)
            for j in range(d):
                layers.append(block(cin, planes, (1 if i == 0 else 2) if j == 0 else 1))
                cin = planes * block.expansion
        self.layers = nn.Sequential(*layers)
        self.depths = list(depths)       # stage boundaries for forward(x, layer)
        self.feat_dim, self.low_dim = cin, low_dim
        if mlp:
            self.fc = nn.Sequential(nn.Linear(cin, cin), nn.ReLU(inplace=True), nn.Linear(cin, low_dim))
        else:
            self.fc = nn.Linear(cin, low_dim)
        # l2norm=False: return the raw fc output -- the contrast head then normalises inside its kernels
        # (MemoryMoCo.forward_loss(..., normalize=True), SURVEY.md 8 f2)
        self.l2norm = True
        self.accepts_s2d = True          # forward() also takes moco_crop_s2d_bf16's 16-channel layout (StemConv)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)

    def freeze(self):
        """A frozen feature extractor for linear evaluation (eval.py:140-146,213): ``eval()``, no parameter requires
        grad, and every BatchNorm is marked frozen.  Under ``torch.no_grad()`` and bf16 autocast (as the training step
        runs the encoders), a frozen model in eval mode runs its BatchNorms on the eval kernels (bn.py), the
        reference's fp32 NCHW [N, 3, H, W] images enter the stem through ``crop_to_s2d_bf16``, and for layer >= 6
        the last block returns the pooled features (so a forward hook on ``layers[-1]`` sees [N, C] there, and
        ``layers`` itself is walked block by block).  ``train()``, grad mode, fp32 without autocast or
        ``bn.set_fused(False)`` run exactly what an unfrozen model runs.  Calling it again also drops the folded
        BatchNorm coefficients (``BatchNormAct2d.folded``), e.g. after weights were written through ``.data``.
        Returns self."""
        self.eval()
        self.requires_grad_(False)
        for m in self.modules():
            if isinstance(m, BatchNormAct2d):
                m.frozen = True
                m._fold_key = m._fold = None
        return self

    def _frozen_active(self):
        """The BatchNorms may take the eval kernels: frozen, eval mode, grad mode off, the fused kernels enabled."""
        bn = self.stem[1]
        return bn_mod._enabled and bn.frozen and not bn.training and not torch.is_grad_enabled()

    def _frozen_input(self, x):
        """Convert the images to the space-to-depth bf16 layout only where the stem convolution computes in bf16
        anyway (bf16 autocast, or bf16 weights): fp32 evaluation keeps the fp32 7x7 convolution."""
        bf16 = ((torch.is_autocast_enabled("cuda") and torch.get_autocast_dtype("cuda") == torch.bfloat16)
                or self.stem[0].weight.dtype == torch.bfloat16)
        return (bf16 and x.is_cuda and x.dim() == 4 and x.shape[1] == 3 and x.shape[2] % 2 == 0
                and x.shape[3] % 2 == 0 and x.dtype in (torch.float32, torch.bfloat16))

    def forward(self, x, layer=7):
        if layer <= 0:
            return x
        frozen = self._frozen_active()
        if frozen and self._frozen_input(x):
            x = crop_to_s2d_bf16(x)                   # StemConv's space-to-depth input, one pass
        conv, bn, _, pool = self.stem                 # index 2 is the Identity placeholder
        x = bn.forward_maxpool(conv(x), pool)
        if layer == 1:
            return x
        if layer >= 6 and not frozen:
            x = torch.flatten(F.adaptive_avg_pool2d(self.layers(x), 1), 1)
        else:
            ends = [sum(self.depths[:i + 1]) for i in range(len(self.depths))]
            last = len(self.layers) - 1
            for i, block in enumerate(self.layers):
                if i == last and layer >= 6:
                    x = block(x, avgpool=True)        # [N, C]: the frozen path never writes the last block's map
                else:
                    x = block(x)
                if i + 1 in ends and layer == 2 + ends.index(i + 1):
                    return x
        if layer == 6:
            return x
        x = self.fc(x).float()
        if not self.l2norm:
            return x
        return x / x.pow(2).sum(1, keepdim=True).sqrt()       # Normalize(power=2), resnet.py:30-33

def resnet18(low_dim=128, width=1, mlp=False):
    return MoCoResNet(_Basic, [2, 2, 2, 2], low_dim, width, mlp)


def resnet34(low_dim=128, width=1, mlp=False):
    return MoCoResNet(_Basic, [3, 4, 6, 3], low_dim, width, mlp)


def resnet50(low_dim=128, width=1, mlp=False):
    return MoCoResNet(_Bottleneck, [3, 4, 6, 3], low_dim, width, mlp)


def has_mlp_head(sd) -> bool:
    """Whether an encoder state_dict (either key naming, ``module.`` prefix optional) carries MoCo v2's MLP head."""
    return any(k.removeprefix("module.").startswith("fc.0.") for k in sd)


def encoder_from_state_dict(sd, arch="resnet50", width=1, low_dim=128):
    """The ``arch`` encoder with the head ``sd`` carries (the MLP head or the bare Linear), ``sd`` loaded into it:
    every driver that builds an encoder for a checkpoint goes through here."""
    sd = from_reference_state_dict(sd)
    model = {"resnet18": resnet18, "resnet34": resnet34, "resnet50": resnet50}[arch](low_dim, width, has_mlp_head(sd))
    model.load_state_dict(sd)
    return model


# ---- checkpoints in the reference's naming ------------------------------------------------------------------------
# The two models have the same state_dict entries in the same order; only the names differ:
#     stem.0.*  <-> conv1.*          stem.1.*  <-> bn1.*
#     layers.<i>.* <-> layer<s>.<j>.*  (block i is block j of stage s)     short.0/1 <-> downsample.0/1
# A stage starts at block 0 and at every later block with a shortcut, so the mapping needs no depths argument.

def _strip_module(sd):
    return {(k[len("module."):] if k.startswith("module.") else k): v for k, v in sd.items()}


def to_reference_state_dict(sd):
    """This package's encoder state_dict (``module.`` prefix optional) -> the reference ResNet's names."""
    sd = _strip_module(sd)
    starts = sorted({int(k.split(".")[1]) for k in sd if k.startswith("layers.") and ".short." in k} | {0})
    out = {}
    for k, v in sd.items():
        parts = k.split(".")
        if parts[0] == "stem":
            k = ".".join([{"0": "conv1", "1": "bn1"}[parts[1]]] + parts[2:])
        elif parts[0] == "layers":
            i = int(parts[1])
            s = sum(1 for b in starts if b <= i)
            j = i - max(b for b in starts if b <= i)
            rest = ["downsample" if p == "short" else p for p in parts[2:]]
            k = ".".join([f"layer{s}", str(j)] + rest)
        out[k] = v
    return out


def from_reference_state_dict(sd):
    """The reference ResNet's state_dict (or a checkpoint's ``model`` entry; ``module.`` prefix optional) -> this
    package's names.  A state_dict already in this package's naming is returned with the prefix stripped."""
    sd = _strip_module(sd)
    if not any(k.startswith("conv1.") for k in sd):
        return sd
    blocks = {}
    for k in sd:
        if k.startswith("layer"):
            s, j = k.split(".")[:2]
            blocks[int(s[len("layer"):])] = max(blocks.get(int(s[len("layer"):]), 0), int(j) + 1)
    first = {s: sum(blocks[t] for t in blocks if t < s) for s in blocks}
    out = {}
    for k, v in sd.items():
        parts = k.split(".")
        if parts[0] in ("conv1", "bn1"):
            k = ".".join(["stem", {"conv1": "0", "bn1": "1"}[parts[0]]] + parts[1:])
        elif parts[0].startswith("layer"):
            i = first[int(parts[0][len("layer"):])] + int(parts[1])
            rest = ["short" if p == "downsample" else p for p in parts[2:]]
            k = ".".join(["layers", str(i)] + rest)
        out[k] = v
    return out
