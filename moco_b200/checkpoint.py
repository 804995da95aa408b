"""Checkpoints in the reference's formats, read and written by both example drivers.

A pre-training checkpoint (train.py:139-172; ``state`` / ``restore``) is a dict with the reference's keys: ``opt``
(the run's arguments), ``model`` (the query encoder in the reference's naming with DistributedDataParallel's
``module.`` prefix), ``model_ema`` (reference naming), ``contrast``, ``optimizer``, ``scheduler`` and ``epoch``.

A classifier checkpoint of the linear evaluation (eval.py:173-185; ``classifier_state`` / ``restore_classifier``) has
eval.py's keys: ``opt``, ``epoch``, ``classifier`` (its ``state_dict`` with the ``module.`` prefix, as eval.py:211
always wraps it in DistributedDataParallel), ``best_acc1`` (a float, in percent), ``optimizer`` and ``scheduler``.

What this module writes holds only tensors and plain Python values: ``opt`` is ``vars(args)`` and ``scheduler`` is
``{"last_epoch": t}``, so it loads under torch.load's default ``weights_only=True`` -- also in the reference's own
``eval.py:load_pretrained``.  ``save`` and ``write_config`` write either kind.

``load`` reads this format and the reference's own ``current.pth``, whose ``opt`` is an ``argparse.Namespace``:
that one class is allow-listed for the weights-only unpickler; nothing else is, and there is no fall-back to
unrestricted unpickling.
"""
from __future__ import annotations

import argparse
import json
import os

import torch

from .encoders import from_reference_state_dict, to_reference_state_dict


def load(path: str) -> dict:
    """The checkpoint at ``path`` on the CPU, unpickled with ``weights_only=True`` and argparse.Namespace allowed."""
    with torch.serialization.safe_globals([argparse.Namespace]):
        return torch.load(path, map_location="cpu", weights_only=True)


def state(args, epoch: int, model, model_ema, contrast, optimizer, scheduler) -> dict:
    """The checkpoint dict of ``epoch`` (``model`` may be wrapped in DistributedDataParallel)."""
    net = model.module if hasattr(model, "module") else model
    return {
        "opt": dict(vars(args)),
        "model": {"module." + k: v for k, v in to_reference_state_dict(net.state_dict()).items()},
        "model_ema": to_reference_state_dict(model_ema.state_dict()),
        "contrast": contrast.state_dict(),
        "optimizer": optimizer.state_dict(),
        "scheduler": {"last_epoch": scheduler.last_epoch},
        "epoch": epoch,
    }


def _save_atomic(obj, path: str) -> None:
    tmp = path + ".tmp"
    torch.save(obj, tmp)
    os.replace(tmp, path)          # an interrupted save leaves the previous file, never a truncated one


def save(ckpt: dict, output_dir: str, save_freq: int) -> None:
    """Write ``current.pth``, and ``ckpt_epoch_{e}.pth`` when e % save_freq == 0 (train.py:155-159), each through
    a temporary file and os.replace.  ``current.pth`` is written at every call, also for a classifier checkpoint,
    which eval.py:244-246 writes only every save_freq epochs: resuming needs the last epoch's."""
    epoch = ckpt["epoch"]
    _save_atomic(ckpt, os.path.join(output_dir, "current.pth"))
    if save_freq > 0 and epoch % save_freq == 0:
        _save_atomic(ckpt, os.path.join(output_dir, f"ckpt_epoch_{epoch}.pth"))


def write_config(args, output_dir: str) -> str:
    """``config.json`` with the run's arguments (train.py:305-309, eval.py:373-377); returns its path."""
    path = os.path.join(output_dir, "config.json")
    with open(path, "w") as f:
        json.dump(vars(args), f, indent=2)
    return path


def restore(ckpt: dict, model, model_ema, contrast, optimizer) -> int:
    """Load a checkpoint of either project into the models (either key naming, ``module.`` optional), the queue
    and the optimizer's momentum; returns the epoch to start from, ``ckpt["epoch"] + 1``.  The scheduler entry is
    not read: the schedule is a closed form of the iteration count, which the caller sets from that epoch."""
    net = model.module if hasattr(model, "module") else model
    net.load_state_dict(from_reference_state_dict(ckpt["model"]))
    model_ema.load_state_dict(from_reference_state_dict(ckpt["model_ema"]))
    contrast.load_state_dict(ckpt["contrast"])
    optimizer.load_state_dict(ckpt["optimizer"])
    return int(ckpt["epoch"]) + 1


def classifier_state(args, epoch: int, classifier, best_acc1: float, optimizer, scheduler) -> dict:
    """The classifier checkpoint of ``epoch`` (``classifier`` may be wrapped in DistributedDataParallel).
    ``best_acc1`` is the best top-1 so far; the reference stores the epoch's own top-1 under that name."""
    net = classifier.module if hasattr(classifier, "module") else classifier
    return {
        "opt": dict(vars(args)),
        "epoch": epoch,
        "classifier": {"module." + k: v for k, v in net.state_dict().items()},
        "best_acc1": float(best_acc1),
        "optimizer": optimizer.state_dict(),
        "scheduler": {"last_epoch": scheduler.last_epoch},
    }


def restore_classifier(ckpt: dict, classifier, optimizer) -> tuple[int, float]:
    """Load a classifier checkpoint of either project (``module.`` optional) into the classifier and the optimizer's
    momentum; returns ``(ckpt["epoch"] + 1, best_acc1)``.  A classifier of another layer, width or class count fails
    with load_state_dict's size-mismatch error.  The reference's ``best_acc1`` may be a tensor, and its scheduler
    entry is not read: the schedule is a closed form of the iteration count, which the caller sets from the epoch."""
    net = classifier.module if hasattr(classifier, "module") else classifier
    net.load_state_dict({k.removeprefix("module."): v for k, v in ckpt["classifier"].items()})
    optimizer.load_state_dict(ckpt["optimizer"])
    return int(ckpt["epoch"]) + 1, float(ckpt["best_acc1"])
