"""Runs the UNMODIFIED reference training loop (``train.train_moco``, train.py:231-293 of bl0/moco) on the host
cores -- TEST/BASELINE INFRASTRUCTURE ONLY (bench.py's ``--impl reference`` arm and ``cpu_baseline`` leg).

The reference sources are the staged copy under ``oracle/_ref/`` (see ``oracle/stage_ref.py``; byte-identical to
/root/reference, git-ignored, shipped to the GPU box with the snapshot).  Nothing of ``moco_b200`` is on this
path: models are the reference's own ``moco.models.resnet``, the head is its ``moco.NCE.MemoryMoCo`` /
``NCESoftmaxLoss``, ShuffleBN its ``DistributedShufle`` over a gloo process group, the optimizer / scheduler /
EMA exactly what ``train.main`` builds (train.py:175-198).

Shims (none touches a reference file):
  1. identity ``torch.Tensor.cuda`` / ``nn.Module.cuda`` -- the reference hard-codes ``.cuda()``
     (Contrast.py:32, util.py:104-108, train.py:253-254);
  2. a stub ``termcolor`` module (moco/logger.py:6 imports it; the package is not installed);
  3. a single-rank ``gloo`` process group in place of ``nccl`` (train.py:300), and ``train.logger`` (a module
     global that only ``__main__`` defines, train.py:304).
``warmup_epoch`` must be >= 1 (lr_scheduler.py:29 divides by it).
"""
from __future__ import annotations

import argparse
import logging
import os
import sys
import tempfile
import time
import types
import warnings

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(HERE, "_ref")


def available() -> bool:
    return os.path.isfile(os.path.join(REF, "train.py")) and os.path.isdir(os.path.join(REF, "moco", "NCE"))


def host_threads() -> int:
    """Threads the CPU arm uses: one per PHYSICAL core the process may run on (what torch picks by itself in a
    clean environment; torchrun exports OMP_NUM_THREADS=1 to its workers, which would otherwise pin the arm to one
    thread, and two oneDNN threads per core only fight over the FMA units)."""
    try:
        allowed = len(os.sched_getaffinity(0))
    except AttributeError:
        allowed = os.cpu_count() or 1
    try:
        import psutil
        phys = psutil.cpu_count(logical=False) or allowed
    except Exception:
        phys = allowed
    return max(1, min(allowed, phys))


_train = None


def _load_reference():
    """Import the staged reference with the three shims applied (idempotent)."""
    global _train
    if _train is not None:
        return _train
    if not available():
        raise RuntimeError("oracle/_ref is not staged: run __graft_entry__.build() where /root/reference exists")
    import torch
    import torch.distributed as dist
    if "termcolor" not in sys.modules:
        stub = types.ModuleType("termcolor")
        stub.colored = lambda s, *a, **k: s
        sys.modules["termcolor"] = stub
    if REF not in sys.path:
        sys.path.insert(0, REF)
    torch.Tensor.cuda = lambda self, *a, **k: self          # the CPU arm stays on the host even on a GPU box
    torch.nn.Module.cuda = lambda self, *a, **k: self
    if not dist.is_initialized():
        store = os.path.join(tempfile.mkdtemp(prefix="moco_ref_pg_"), "store")
        dist.init_process_group("gloo", init_method=f"file://{store}", rank=0, world_size=1)
    import train  # noqa: E402  (oracle/_ref/train.py == the reference's train.py)
    train.logger = logging.getLogger("moco_ref")
    train.logger.setLevel(logging.WARNING)
    _train = train
    return train


def _args(batch: int, K: int, T: float, steps_per_epoch: int):
    """The argparse namespace train.main / train_moco / get_scheduler read (defaults of train.py:35-84)."""
    return argparse.Namespace(
        batch_size=batch, nce_k=K, nce_t=T, alpha=0.999, base_learning_rate=0.1, lr_scheduler="cosine",
        warmup_epoch=1, warmup_multiplier=100, lr_decay_epochs=[120, 160, 200], lr_decay_rate=0.1,
        weight_decay=1e-4, momentum=0.9, amp_opt_level="O0", epochs=200, start_epoch=1, print_freq=10 ** 9,
        local_rank=0, model_width=1)


class ReferenceJob:
    """What ``train.main`` builds (train.py:175-198), with the backbone selectable (train.py:49,129 only wires
    resnet50; BASELINE configs[0] is ResNet-18) and synthetic two-crop batches (dataset.py:31-33 layout)."""

    def __init__(self, arch: str, feat_dim: int, K: int, T: float, batch: int, n_batches: int, seed: int = 0):
        import torch
        import torch.distributed as dist
        from torch.nn.parallel import DistributedDataParallel
        train = _load_reference()
        from moco.NCE import MemoryMoCo, NCESoftmaxLoss
        from moco.lr_scheduler import get_scheduler
        from moco.models import resnet as ref_resnet
        from moco.util import moment_update
        self.train = train
        self.args = _args(batch, K, T, n_batches)
        torch.manual_seed(seed)
        ctor = getattr(ref_resnet, arch)
        model, model_ema = ctor(low_dim=feat_dim).cuda(), ctor(low_dim=feat_dim).cuda()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            moment_update(model, model_ema, 0)                                   # train.py:133
        self.contrast = MemoryMoCo(feat_dim, K, T).cuda()                        # train.py:181
        self.criterion = NCESoftmaxLoss().cuda()
        self.optimizer = torch.optim.SGD(model.parameters(),                     # train.py:183-186
                                         lr=batch * dist.get_world_size() / 256 * self.args.base_learning_rate,
                                         momentum=self.args.momentum, weight_decay=self.args.weight_decay)
        self.scheduler = get_scheduler(self.optimizer, max(1, n_batches), self.args)
        self.model = DistributedDataParallel(model, broadcast_buffers=False)     # train.py:198 (CPU: no device_ids)
        self.model_ema = model_ema
        g = torch.Generator().manual_seed(1234)
        self.batch = torch.randn(batch, 6, 224, 224, generator=g)
        self.epoch = 1

    def run(self, n_batches: int):
        """One call of the reference's train_moco over `n_batches` synthetic batches; returns (seconds, loss, prob)."""
        loader = [(self.batch, None)] * n_batches
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")            # deprecated add_(scalar, tensor) in util.py:127
            t0 = time.perf_counter()
            loss, prob = self.train.train_moco(self.epoch, loader, self.model, self.model_ema, self.contrast,
                                               self.criterion, self.optimizer, self.scheduler, self.args)
            dt = time.perf_counter() - t0
        return dt, float(loss), float(prob)


def time_reference(arch: str, feat_dim: int, K: int, T: float, batch: int, steps: int, warmup: int,
                   budget_s: float = 120.0):
    """images/sec of the unmodified reference step on the host cores: `warmup` untimed + `steps` timed batches of
    `batch` synthetic images.  `steps` is cut (never below 3) only if the warm-up shows the budget would be blown."""
    import torch
    threads = host_threads()
    torch.set_num_threads(threads)
    job = ReferenceJob(arch, feat_dim, K, T, batch, warmup + steps)
    w = max(1, warmup)
    dt_w, _, _ = job.run(w)
    per = dt_w / w
    steps = max(3, min(steps, int(budget_s / max(per, 1e-3))))
    dt, loss, prob = job.run(steps)
    return {"images_per_s": batch * steps / dt, "ms_per_step": dt / steps * 1e3, "steps": steps, "warmup": w,
            "batch": batch, "loss": loss, "prob": prob, "threads": threads, "arch": arch, "K": K,
            "feat_dim": feat_dim, "index": int(job.contrast.index)}


if __name__ == "__main__":
    import json
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="resnet18")
    ap.add_argument("--feat-dim", type=int, default=128)
    ap.add_argument("--nce-k", type=int, default=1024)
    ap.add_argument("--nce-t", type=float, default=0.07)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    print(json.dumps(time_reference(a.arch, a.feat_dim, a.nce_k, a.nce_t, a.batch, a.steps, a.warmup)))
