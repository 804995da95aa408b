"""The linear classifier of the reference's linear evaluation (moco/models/LinearModel.py), with the same module names
and ``state_dict`` keys -- including the reference's ``classifier.LiniearClassifier.*`` spelling -- so that
classifier checkpoints move between the two projects unchanged.

The features it takes are those of ``MoCoResNet.forward(x, layer)`` for layers 2..6 of a ResNet-50 (2048 * width
channels at layer 6).  Layer 1 is kept as the reference defines it, for 128 * width channels, but the stem's output
has 64 in both models, so a layer-1 classifier cannot take a ResNet-50's layer-1 features (nor can the reference's).
Flattening follows the logical NCHW order of the reference's ``Flatten`` (``feat.view(N, -1)``) also when the
features are channels_last, where a view is not possible and ``reshape`` copies.
"""
from __future__ import annotations

from torch import nn

# layer -> (pool size, channels at width 1) of a ResNet-50 (LinearModel.py:17-40)
_LAYERS = {1: (8, 128), 2: (6, 256), 3: (4, 512), 4: (3, 1024), 5: (7, 2048), 6: (1, 2048)}


class Flatten(nn.Module):
    def forward(self, feat):
        return feat.reshape(feat.size(0), -1)


class LinearClassifierResNet(nn.Module):
    def __init__(self, layer=6, n_label=1000, pool_type="avg", width=1):
        super().__init__()
        if layer not in _LAYERS:
            raise NotImplementedError(f"layer not supported: {layer}")
        pool_size, channels = _LAYERS[layer]
        self.classifier = nn.Sequential()
        if layer < 5:
            if pool_type == "max":
                self.classifier.add_module("MaxPool", nn.AdaptiveMaxPool2d((pool_size, pool_size)))
            elif pool_type == "avg":
                self.classifier.add_module("AvgPool", nn.AdaptiveAvgPool2d((pool_size, pool_size)))
        self.classifier.add_module("Flatten", Flatten())
        self.classifier.add_module("LiniearClassifier", nn.Linear(channels * width * pool_size * pool_size, n_label))
        for m in self.modules():
            if isinstance(m, nn.Linear):
                m.weight.data.normal_(0, 0.01)
                m.bias.data.fill_(0.0)

    def forward(self, x):
        return self.classifier(x)
