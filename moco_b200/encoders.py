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

from .bn import BatchNormAct2d, MaxPool3x3s2


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

    def forward(self, x):
        y = self.bn1(self.conv1(x))
        if self.short is None:
            return self.bn2(self.conv2(y), x)
        return self.bn2(self.conv2(y), self.short[0](x), shortcut_bn=self.short[1])   # one BN group for both


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

    def forward(self, x):
        y = self.bn1(self.conv1(x))
        y = self.bn2(self.conv2(y))
        if self.short is None:
            return self.bn3(self.conv3(y), x)
        return self.bn3(self.conv3(y), self.short[0](x), shortcut_bn=self.short[1])   # one BN group for both


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
    """ResNet trunk -> global average pool -> fc(low_dim) -> L2 normalise."""

    def __init__(self, block, depths, low_dim=128, width=1):
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

    def forward(self, x):
        conv, bn, _, pool = self.stem                 # index 2 is the Identity placeholder
        x = self.layers(bn.forward_maxpool(conv(x), pool))
        x = torch.flatten(F.adaptive_avg_pool2d(x, 1), 1)
        x = self.fc(x).float()
        if not self.l2norm:
            return x
        return x / x.pow(2).sum(1, keepdim=True).sqrt()       # Normalize(power=2), resnet.py:30-33


def resnet18(low_dim=128, width=1):
    return MoCoResNet(_Basic, [2, 2, 2, 2], low_dim, width)


def resnet34(low_dim=128, width=1):
    return MoCoResNet(_Basic, [3, 4, 6, 3], low_dim, width)


def resnet50(low_dim=128, width=1):
    return MoCoResNet(_Bottleneck, [3, 4, 6, 3], low_dim, width)
