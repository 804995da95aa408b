"""The linear classifier of the reference's linear evaluation (moco/models/LinearModel.py), with the same module names
and ``state_dict`` keys -- including the reference's ``classifier.LiniearClassifier.*`` spelling -- so that
classifier checkpoints move between the two projects unchanged.

The features it takes are those of ``MoCoResNet.forward(x, layer)`` for layers 2..6 of a ResNet-50 (2048 * width
channels at layer 6).  Layer 1 is kept as the reference defines it, for 128 * width channels, but the stem's output
has 64 in both models, so a layer-1 classifier cannot take a ResNet-50's layer-1 features (nor can the reference's).
Flattening follows the logical NCHW order of the reference's ``Flatten`` (``feat.view(N, -1)``) also when the
features are channels_last, where a view is not possible and ``reshape`` copies.

Also the rest of eval.py's recipe around the classifier:

* ``get_scheduler``: the per-iteration learning-rate schedule of moco/lr_scheduler.py -- a linear warm-up from
  lr / multiplier to lr, then cosine annealing or step decay -- computed from its closed form at every step.
* Exact validation: ``ShardSampler`` gives rank r the samples range(r, n, world), with no padding, ``val_totals``
  sums one batch's loss x size, top-1 / top-5 correct counts and size, and ``finish_validation`` adds the ranks'
  sums with one all_reduce.  The accuracy is then over exactly the n samples of the validation set.  The reference's
  DistributedSampler pads the set by repeating samples until it divides by the world size, and its ``validate``
  averages per-batch, per-rank means, so its figure can differ from this one in the last digits.
"""
from __future__ import annotations

import bisect
import math

import torch
from torch import nn
from torch.optim.lr_scheduler import LRScheduler

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


class WarmupSchedule(LRScheduler):
    """lr(t) of iteration t (``step()`` once per iteration, after ``optimizer.step()``) for each group's initial lr:
    base / m * ((m - 1) * t / W + 1) while t <= W, then ``after(base, t - W)``.  W = 0 means no warm-up."""

    def __init__(self, optimizer, multiplier, warmup_iters, after, last_epoch=-1):
        if multiplier <= 1.0:
            raise ValueError("warmup multiplier should be greater than 1")
        self.multiplier = multiplier
        self.warmup_iters = int(warmup_iters)
        self.after = after
        super().__init__(optimizer, last_epoch)

    def lr_at(self, base: float, t: int) -> float:
        m, w = self.multiplier, self.warmup_iters
        if w > 0 and t <= w:
            return base / m * ((m - 1.0) * t / w + 1.0)
        return self.after(base, t - w)

    def get_lr(self):
        return [self.lr_at(base, self.last_epoch) for base in self.base_lrs]


def get_scheduler(optimizer, n_iter_per_epoch: int, epochs: int, kind: str = "cosine", warmup_epoch: int = 5,
                  warmup_multiplier: float = 100, decay_epochs=(30, 60, 90), decay_rate: float = 0.1) -> WarmupSchedule:
    """eval.py's schedule (``--lr-scheduler``, ``--warmup-epoch``, ``--warmup-multiplier``, ``--lr-decay-epochs``,
    ``--lr-decay-rate``), per iteration.  Warm-up: linear from lr / warmup_multiplier to lr over
    warmup_epoch * n_iter_per_epoch iterations.  Then ``kind="cosine"``: cosine annealing to 1e-6 over the remaining
    (epochs - warmup_epoch) * n_iter_per_epoch iterations; ``kind="step"``: lr * decay_rate ** k after the k-th of the
    milestones (m - warmup_epoch) * n_iter_per_epoch, counted from the end of the warm-up.  warmup_multiplier <= 1
    raises ValueError, as the reference does.  warmup_epoch = 0 starts the decay at the first iteration, where the
    reference divides by zero."""
    warmup = warmup_epoch * n_iter_per_epoch
    if kind == "cosine":
        eta_min, t_max = 1e-6, max((epochs - warmup_epoch) * n_iter_per_epoch, 1)

        def after(base, t):
            return eta_min + (base - eta_min) * (1 + math.cos(math.pi * t / t_max)) / 2
    elif kind == "step":
        milestones = sorted((m - warmup_epoch) * n_iter_per_epoch for m in decay_epochs)

        def after(base, t):
            return base * decay_rate ** bisect.bisect_right(milestones, t)
    else:
        raise ValueError(f"scheduler {kind!r} not supported (cosine or step)")
    return WarmupSchedule(optimizer, warmup_multiplier, warmup, after)


class ShardSampler(torch.utils.data.Sampler):
    """The validation split of rank ``rank`` out of ``world``: indices range(rank, n, world), in order, no padding."""

    def __init__(self, n: int, rank: int = 0, world: int = 1):
        if not 0 <= rank < world:
            raise ValueError(f"rank {rank} outside world {world}")
        self.indices = range(rank, n, world)

    def __iter__(self):
        return iter(self.indices)

    def __len__(self):
        return len(self.indices)


def val_totals(output: torch.Tensor, target: torch.Tensor, loss: torch.Tensor, topk=(1, 5)) -> torch.Tensor:
    """float64 [2 + len(topk)] sums of one validation batch: loss * batch size, the top-k correct counts (top-k as
    moco/util.py:accuracy takes it; k is capped at the number of classes, where every sample is correct) and the
    batch size.  ``loss`` is the batch's mean loss."""
    n = target.shape[0]
    maxk = min(max(topk), output.shape[1])
    _, pred = output.topk(maxk, 1, True, True)
    correct = pred.t().eq(target.view(1, -1).expand(maxk, n))
    counts = [correct[:k].reshape(-1).sum() for k in topk]
    return torch.stack([loss.detach().double() * n] + [c.double() for c in counts]
                       + [torch.tensor(float(n), dtype=torch.float64, device=output.device)])


def finish_validation(totals: torch.Tensor, n_expected: int, group=None) -> dict:
    """The ranks' ``val_totals`` sums added by one all_reduce (when a process group is initialised) -> mean loss and
    top-k accuracy in percent over all samples.  Asserts that exactly ``n_expected`` samples were counted."""
    import torch.distributed as dist
    totals = totals.clone()
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(totals, group=group)
    t = totals.tolist()
    n = int(round(t[-1]))
    assert n == n_expected, f"validation counted {n} samples, the set has {n_expected}"
    return {"n": n, "loss": t[0] / max(n, 1), "acc": [100.0 * c / max(n, 1) for c in t[1:-1]]}
