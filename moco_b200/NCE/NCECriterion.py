"""NCESoftmaxLoss -- drop-in for moco/NCE/NCECriterion.py:5-13 of bl0/moco.

``forward(x)`` is CrossEntropyLoss(x, label 0) with mean reduction.  When ``x`` is
the tensor ``moco_b200.NCE.MemoryMoCo.forward`` just returned (unmodified), the
loss was already produced by the fused tensor-core kernel (with its own backward to
q), so it is returned as is and the [N, K+1] logits are not read again.  For any
other input the definition is evaluated directly.
"""
import torch
from torch import nn


class NCESoftmaxLoss(nn.Module):
    """Softmax cross-entropy loss (a.k.a., info-NCE loss in CPC paper)"""

    def __init__(self):
        super().__init__()

    def forward(self, x):
        fused = getattr(x, "_moco_fused", None)
        if fused is not None and fused[2] == x._version:
            return fused[0]
        # generic definition: mean_i( logsumexp_j x_ij - x_i0 )   (NCECriterion.py:11-13)
        return (torch.logsumexp(x.float(), dim=1) - x[:, 0].float()).mean()


def fused_prob(x):
    """``softmax(x, 1)[:, 0].mean()`` (train.py:264) without re-reading the logits when ``x`` came
    from MemoryMoCo.forward; falls back to the definition otherwise."""
    fused = getattr(x, "_moco_fused", None)
    if fused is not None and fused[2] == x._version:
        return fused[1]
    return torch.softmax(x.float(), dim=1)[:, 0].mean()
