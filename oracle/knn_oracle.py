"""Float64 numpy oracle of the weighted kNN contract (include/moco_b200.h: moco_knn; TEST INFRASTRUCTURE ONLY).

The reference has no kNN; the vote is lemniscate.pytorch's (weights exp(s / T) summed per class of the k nearest
bank rows), with its ties defined: the neighbours are the first k rows under (s descending, j ascending), the
predictions the classes under (score descending, class ascending).  Everything here is float64 and sequential, so on
inputs whose dot products are exact in fp32 the neighbours equal the kernel's exactly, and the scores differ from its
fp32 ones by rounding only.
"""
from __future__ import annotations

import numpy as np


def similarities(q: np.ndarray, bank: np.ndarray) -> np.ndarray:
    """s[i, j] = q_i . bank_j in float64 (the inputs as given: pass bf16-representable values)."""
    return np.asarray(q, np.float64) @ np.asarray(bank, np.float64).T


def knn(q: np.ndarray, bank: np.ndarray, labels: np.ndarray, k: int, t: float, n_classes: int) -> dict:
    """``idx`` int64 [Nq, k] and ``sims`` [Nq, k]: N(i) in order; ``scores`` [Nq, n_classes]; ``pred`` int64
    [Nq, 5] (-1 past n_classes) and ``top`` [Nq, 5] their scores."""
    s = similarities(q, bank)
    nq, nb = s.shape
    labels = np.asarray(labels, np.int64)
    idx = np.empty((nq, k), np.int64)
    sims = np.empty((nq, k))
    scores = np.zeros((nq, n_classes))
    pred = np.full((nq, 5), -1, np.int64)
    top = np.zeros((nq, 5))
    j = np.arange(nb)
    for i in range(nq):
        order = np.lexsort((j, -s[i]))[:k]                  # primary -s (s descending), then j ascending
        idx[i], sims[i] = order, s[i, order]
        w = np.exp((sims[i] - sims[i, 0]) / t)
        for r in range(k):                                   # N(i)'s order
            scores[i, labels[order[r]]] += w[r]
        c = np.lexsort((np.arange(n_classes), -scores[i]))[:5]
        pred[i, :len(c)], top[i, :len(c)] = c, scores[i, c]
    return {"idx": idx, "sims": sims, "scores": scores, "pred": pred, "top": top}


def ambiguous(scores: np.ndarray, rtol: float) -> np.ndarray:
    """bool [Nq]: rows where two neighbouring class scores among the six best differ, but by at most rtol times the
    larger, or lie where fp32 is subnormal (< 2^-126), so an fp32 vote may order them either way.  Equal scores are
    not: both sides add the same terms in the same order, and the class decides."""
    srt = -np.sort(-scores, axis=1)[:, :6]
    hi, lo = srt[:, :-1], srt[:, 1:]
    close = (hi - lo <= rtol * hi) | (hi < 2.0 ** -126)
    return ((hi > lo) & close).any(axis=1)
