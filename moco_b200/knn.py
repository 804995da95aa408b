"""Weighted k-nearest-neighbour evaluation of a frozen encoder (INTEGRATION.md §7): the check of instance
discrimination (lemniscate.pytorch, whose NCE code the reference took) that needs one forward pass over the train and
val sets and no training.

* ``build_bank``: the L2-normalised features of a whole dataset, bf16 [Nb, C], with int32 labels, in dataset order
  whatever the world size.
* ``knn_predict``: the top-5 classes of each query by a weighted vote of its k nearest bank rows, on ``moco_knn``
  (csrc/knn_sm90.cu), which never stores the similarity matrix.
* ``knn_evaluate``: top-1 / top-5 accuracy over a validation loader, counted exactly over its dataset.
* ``reference_knn``: the same contract in plain torch (``mm``, a sort in the contract's order, the vote), the readable
  statement of it and the oracle of the larger tests.

The contract (include/moco_b200.h, moco_knn): s(i, j) = q_i . bank_j in fp32; the neighbours N(i) are the first k rows
under (s descending, j ascending); score(i, c) = sum over N(i) with label c of exp((s - s_max) / T), added in N(i)'s
order; the predictions are the classes under (score descending, class ascending).
"""
from __future__ import annotations

import ctypes
from typing import NamedTuple

import torch

from . import _lib

MAX_QUERIES = 1024                 # queries per moco_knn call


class KnnResult(NamedTuple):
    pred: torch.Tensor             # int64 [Nq, 5], -1 past n_classes
    scores: torch.Tensor           # fp32 [Nq, 5]
    indices: torch.Tensor | None   # int64 [Nq, k], N(i) in order
    sims: torch.Tensor | None      # fp32 [Nq, k]
    correct: torch.Tensor | None   # int64 [2]: top-1 and top-5 hits, given targets


def _capacity(nb: int, k: int) -> int:
    """The first try's candidates per query: spread similarities need a few times k (INTEGRATION.md §7)."""
    return min(nb, max(16 * k, 8192))


def _knn_chunk(bank, labels, q, k, inv_t, n_classes, targets, want_neighbors, capacity):
    lib = _lib.load()
    nq, c = q.shape
    nb = bank.shape[0]
    dev = q.device
    top5 = torch.empty(nq, 5, dtype=torch.int32, device=dev)
    scores = torch.empty(nq, 5, dtype=torch.float32, device=dev)
    idx = torch.empty(nq, k, dtype=torch.int32, device=dev) if want_neighbors else None
    sims = torch.empty(nq, k, dtype=torch.float32, device=dev) if want_neighbors else None
    correct = torch.empty(2, dtype=torch.int32, device=dev) if targets is not None else None
    ptr = lambda t: None if t is None else t.data_ptr()
    need = ctypes.c_int64(0)
    for attempt in range(2):
        nbytes = lib.moco_knn_workspace_bytes(nq, nb, capacity)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        rc = lib.moco_knn(q.data_ptr(), bank.data_ptr(), labels.data_ptr(), nq, nb, c, k, inv_t, n_classes,
                          ptr(targets), top5.data_ptr(), scores.data_ptr(), ptr(idx), ptr(sims), ptr(correct),
                          ws.data_ptr(), nbytes, ctypes.byref(need), _lib.cur_stream())
        if rc != _lib.ERR_CAPACITY or attempt == 1:
            break
        capacity = int(need.value)             # the same inputs give the same candidates: one rerun suffices
    _lib.check(rc, "moco_knn")
    return top5, scores, idx, sims, correct


def knn_predict(bank: torch.Tensor, labels: torch.Tensor, q: torch.Tensor, k: int = 200, t: float = 0.07,
                n_classes: int | None = None, targets: torch.Tensor | None = None, return_neighbors: bool = False,
                capacity: int | None = None) -> KnnResult:
    """The top-5 classes of each row of q (bf16 or fp32 [Nq, C], rounded to bf16) by its k nearest rows of ``bank``
    (bf16 [Nb, C]) with ``labels`` (int32 [Nb]), weighted exp(s / t).  n_classes defaults to labels.max() + 1.
    targets (int [Nq]): also count the top-1 / top-5 hits.  return_neighbors: also N(i) and its similarities.
    capacity: the first try's candidates per query (a test knob; a query with more makes it retry once with what
    it needs).  Runs moco_knn on chunks of up to 1024 queries."""
    _lib.require_cuda(bank, labels, q, targets)
    if bank.dtype != torch.bfloat16 or bank.dim() != 2:
        raise TypeError("knn_predict: bank must be bf16 [Nb, C]")
    if labels.dtype != torch.int32 or labels.shape != (bank.shape[0],):
        raise TypeError("knn_predict: labels must be int32 [Nb]")
    if q.dim() != 2 or q.shape[1] != bank.shape[1]:
        raise ValueError(f"knn_predict: q {tuple(q.shape)} does not match the bank's C = {bank.shape[1]}")
    if not t > 0:
        raise ValueError("knn_predict: t must be > 0")
    bank = bank.contiguous()
    labels = labels.contiguous()
    q = q.to(torch.bfloat16).contiguous()
    if n_classes is None:
        n_classes = int(labels.max()) + 1
    if targets is not None:
        targets = targets.to(device=q.device, dtype=torch.int32).contiguous()
    if capacity is None:
        capacity = _capacity(bank.shape[0], k)
    capacity = max(min(capacity, bank.shape[0]), k)
    parts = []
    for s in range(0, q.shape[0], MAX_QUERIES):
        e = min(s + MAX_QUERIES, q.shape[0])
        parts.append(_knn_chunk(bank, labels, q[s:e], k, 1.0 / t, n_classes,
                                None if targets is None else targets[s:e], return_neighbors, capacity))
    cat = lambda i: None if parts[0][i] is None else torch.cat([p[i] for p in parts])
    correct = None if targets is None else torch.stack([p[4].long() for p in parts]).sum(0)
    idx = cat(2)
    return KnnResult(cat(0).long(), cat(1), None if idx is None else idx.long(), cat(3), correct)


def reference_knn(bank: torch.Tensor, labels: torch.Tensor, q: torch.Tensor, k: int = 200, t: float = 0.07,
                  n_classes: int | None = None) -> KnnResult:
    """The contract in torch, on any device: fp32 similarities of the bf16 rows, a stable sort that takes (s
    descending, j ascending), the first k, then each rank's weight added to its class in rank order."""
    labels = labels.long()
    if n_classes is None:
        n_classes = int(labels.max()) + 1
    s = q.to(torch.bfloat16).float() @ bank.float().t()
    s = s + 0.0                                                    # -0 is +0, as in the kernel's order
    sims, idx = torch.sort(s, dim=1, descending=True, stable=True)  # ties keep j ascending
    sims, idx = sims[:, :k].contiguous(), idx[:, :k].contiguous()
    w = torch.exp((sims - sims[:, :1]) * (1.0 / t))
    lab = labels[idx]
    score = torch.zeros(q.shape[0], n_classes, dtype=torch.float32, device=q.device)
    for r in range(k):                                             # fp32, N(i)'s order
        score.scatter_add_(1, lab[:, r:r + 1], w[:, r:r + 1])
    order = torch.sort(score, dim=1, descending=True, stable=True).indices[:, :5]   # ties: class ascending
    top = torch.gather(score, 1, order)
    if n_classes < 5:
        pad = 5 - n_classes
        order = torch.cat([order, order.new_full((q.shape[0], pad), -1)], 1)
        top = torch.cat([top, top.new_zeros(q.shape[0], pad)], 1)
    return KnnResult(order, top, idx, sims, None)


def _features(model, x, layer):
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        f = model(x, layer).float()
    if layer == 6:                                                 # layer 7 is normalised by the model
        f = f / f.pow(2).sum(1, keepdim=True).sqrt()
    return f


def build_bank(model, loader, layer: int = 7, device=None) -> tuple[torch.Tensor, torch.Tensor]:
    """(bank bf16 [n, C], labels int32 [n]) of ``loader.dataset``, n = len(loader.dataset), in dataset order.  The
    loader yields ``augment.ImageFolderEval(train=False)`` batches; with a process group of world w > 1 its sampler is
    ``linear_eval.ShardSampler(n, rank, w)``, and one all-gather gives every rank the whole bank.  Layer 7: the fc
    output; 6: the pooled features, L2-normalised here.  The model is run frozen (``freeze()`` first)."""
    import torch.distributed as dist
    from . import augment as A
    if layer not in (6, 7):
        raise ValueError(f"build_bank: layer {layer} (6 or 7)")
    if device is None:
        device = next(model.parameters()).device
    n = len(loader.dataset)
    feats, labs = [], []
    for b in loader:
        x = A.resize_center_crops(b, dtype=torch.bfloat16, device=device)
        feats.append(_features(model, x, layer).bfloat16())
        labs.append(b[2].to(device, torch.int32))
    dim = model.fc.out_features if layer == 7 else model.fc.in_features   # also for a rank with no samples
    f = torch.cat(feats) if feats else torch.empty(0, dim, dtype=torch.bfloat16, device=device)
    lab = torch.cat(labs) if labs else torch.empty(0, dtype=torch.int32, device=device)
    world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    if world == 1:
        assert f.shape[0] == n, f"the loader gave {f.shape[0]} samples, the dataset has {n}"
        return f.contiguous(), lab.contiguous()
    per = (n + world - 1) // world                                 # rank r holds r, r + w, ...: at most `per` rows
    fp = torch.zeros(per, f.shape[1], dtype=f.dtype, device=device)
    lp = torch.zeros(per, dtype=torch.int32, device=device)
    fp[:f.shape[0]] = f
    lp[:lab.shape[0]] = lab
    fa = torch.empty(world, per, f.shape[1], dtype=f.dtype, device=device)
    la = torch.empty(world, per, dtype=torch.int32, device=device)
    dist.all_gather_into_tensor(fa, fp)
    dist.all_gather_into_tensor(la, lp)
    bank = fa.transpose(0, 1).reshape(per * world, f.shape[1])[:n]   # row r + w m of the dataset is rank r's m-th
    return bank.contiguous(), la.t().reshape(-1)[:n].contiguous()


def knn_evaluate(model, bank: torch.Tensor, labels: torch.Tensor, val_loader, k: int = 200, t: float = 0.07,
                 layer: int = 7, n_classes: int | None = None, device=None) -> dict:
    """Top-1 / top-5 kNN accuracy over ``val_loader`` (``ImageFolderEval(train=False)`` batches, with
    ``linear_eval.ShardSampler`` at world > 1): each rank's hits in ``linear_eval.val_totals``' layout (no loss),
    reduced by ``finish_validation``, which asserts that exactly len(val_loader.dataset) samples were counted."""
    from . import augment as A
    from .linear_eval import finish_validation
    if device is None:
        device = bank.device
    if n_classes is None:
        n_classes = int(labels.max()) + 1
    totals = torch.zeros(4, dtype=torch.float64, device=device)   # loss * n, top-1, top-5, n
    for b in val_loader:
        x = A.resize_center_crops(b, dtype=torch.bfloat16, device=device)
        y = b[2].to(device)
        r = knn_predict(bank, labels, _features(model, x, layer), k, t, n_classes, targets=y)
        totals[1:3] += r.correct.double()
        totals[3] += y.shape[0]
    return finish_validation(totals, len(val_loader.dataset))
