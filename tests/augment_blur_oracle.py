"""An exact numpy restatement of moco_augment_crops_blur (include/moco_b200.h), written from the header's contract.

It builds on oracle/augment_oracle.py, which restates moco_augment_crops and is used here unchanged: its tap geometry,
resample, grayscale, blend, hue round trip and contrast-mean order are those of the blur entry point too.  This module
adds the two steps the 32-word records bring:
  * ``gray_late``: the grayscale runs after the jitter instead of before it (the contrast mean is still the mean
    grayscale of the crop as it stands before the contrast op);
  * ``blur``: the full 1-D kernel k [2h + 1] (per crop or shared), after the pointwise ops and before the flip: with
    reflect padding of h, t = sum_j k[j] * s(reflect(y - h + j), x) for j = 0 .. 2h, then out = sum_j k[j] *
    t(y, reflect(x - h + j)), each sum started from 0 in tap order, every product and addition one float32 operation.
``exact=False`` is the high-precision reference, as in oracle/augment_oracle.py: the same float32 geometry, constants
and blur weights, every other operation in float64.

``mutant`` names a deliberately wrong variant (BLUR_MUTANTS); the tests use them to show that a case table catches
such errors.  None is the contract.
"""
from __future__ import annotations

import numpy as np

from oracle import augment_oracle as O

F32, F64 = np.float32, np.float64
GRAY, FLIP, JITTER = O.GRAY, O.FLIP, O.JITTER

# the last two change rounding only: the blur commutes with the flip in exact arithmetic (its taps are symmetric), and
# the 2-D product kernel is the same sum in another order
BLUR_MUTANTS = ("blur_zero_pad", "blur_replicate_pad", "gray_before_jitter", "blur_drop_outer_tap",
                "blur_after_flip", "blur_2d_weights")
BLUR_SEMANTIC_MUTANTS = BLUR_MUTANTS[:4]


def _gray3(r, g, b):
    lum = O.gray(r, g, b)
    return lum, lum, lum


def _pointwise(r, g, b, flags, order, factors, mean, gray_late):
    """The ops after the resample; with mean None, stop before the contrast op and return its input."""
    ft = r.dtype.type
    if flags & GRAY and not gray_late:
        r, g, b = _gray3(r, g, b)
    if flags & JITTER:
        f = factors.astype(ft)[:, :, None, None]                     # [N, 4, 1, 1]
        fm = (1.0 - factors.astype(F64)).astype(F32).astype(ft)[:, :, None, None]
        for k in range(4):
            op = (order >> (2 * k)) & 3
            fk, fmk = f[:, op], fm[:, op]
            if op == 0:
                zero = np.zeros_like(r)
                r, g, b = (O._blend(x, zero, fk, fmk) for x in (r, g, b))
            elif op == 1:
                if mean is None:
                    return r, g, b
                m = mean.astype(ft)[:, None, None]
                r, g, b = (O._blend(x, m, fk, fmk) for x in (r, g, b))
            elif op == 2:
                lum = O.gray(r, g, b)
                r, g, b = (O._blend(x, lum, fk, fmk) for x in (r, g, b))
            else:
                r, g, b = O.hue_shift(r, g, b, fk)
    if flags & GRAY and gray_late:
        r, g, b = _gray3(r, g, b)
    return r, g, b


def reflect(i, n):
    """Reflect padding's source index of index i (no edge repeat): -i -> i, n - 1 + i -> n - 1 - i."""
    i = np.abs(i)
    return np.where(i >= n, 2 * (n - 1) - i, i)


def blur(x, k, mutant=None):
    """x [N, 3, H, W] (float32 or float64), k [N, 2h + 1] in the same dtype: the separable blur in the contract's
    order, vertical pass then horizontal pass, each in tap order."""
    n, _, H, W = x.shape
    taps = k.shape[1]
    h = taps // 2
    if mutant == "blur_drop_outer_tap":
        k = k.copy()
        k[:, 0] = k[:, -1] = 0
    if mutant in ("blur_zero_pad", "blur_replicate_pad"):             # pad explicitly; indices shift by h
        x = np.pad(x, ((0, 0), (0, 0), (h, h), (h, h)), mode="constant" if mutant == "blur_zero_pad" else "edge")
        rows = lambda j: np.arange(H) + j
        cols = lambda j: np.arange(W) + j
    else:
        rows = lambda j: reflect(np.arange(H) - h + j, H)
        cols = lambda j: reflect(np.arange(W) - h + j, W)
    kk = k[:, :, None, None, None]
    if mutant == "blur_2d_weights":
        k2 = (k[:, :, None] * k[:, None, :])[:, :, :, None, None, None]
        out = np.zeros((n, 3, H, W), x.dtype)
        for a in range(taps):
            for b in range(taps):
                out = out + k2[:, a, b] * x[:, :, rows(a)][:, :, :, cols(b)]
        return out
    t = np.zeros((n, 3, H, x.shape[3]), x.dtype)
    for j in range(taps):
        t = t + kk[:, j] * x[:, :, rows(j)]
    out = np.zeros((n, 3, H, W), x.dtype)
    for j in range(taps):
        out = out + kk[:, j] * t[:, :, :, cols(j)]
    return out


def augment(box, out_h, out_w, flags, order, factors, norm, exact=True, mutant=None, gray_late=False, blur_k=None):
    """moco_augment_crops_blur on N crops of one geometry.  box: uint8 [N, hh, ww, 3], each crop's box cut from its
    image; factors: float32 [N, 4]; ``gray_late`` the record's gray_after_jitter; ``blur_k`` None (no blur) or float32
    [2h + 1] / [N, 2h + 1], the full 1-D kernel.  Returns (out [N, 3, out_h, out_w], crop means [N], 0 where jitter
    is off), float32 when exact else float64."""
    box = np.asarray(box, np.uint8)
    factors = np.asarray(factors, F32).reshape(-1, 4)
    hh, ww = box.shape[1], box.shape[2]
    ty, tx = O.Taps(np.arange(out_h), hh, out_h), O.Taps(np.arange(out_w), ww, out_w)
    cw = O.chunk_width(ww, out_w, out_w)
    r, g, b = O._resample(box, ty, tx, exact, None, cw)
    ft = F32 if exact else F64
    gray_late = gray_late and mutant != "gray_before_jitter"
    mean = np.zeros(box.shape[0], ft)
    if flags & JITTER:
        lum = O.gray(*_pointwise(r, g, b, flags, order, factors, None, gray_late))
        mean = O.contrast_mean(lum, cw) if exact else lum.mean(axis=(1, 2))
    r, g, b = _pointwise(r, g, b, flags, order, factors, mean, gray_late)
    x = np.stack([r, g, b], axis=1)                                   # [N, 3, H, W]
    k = None
    if blur_k is not None:
        k32 = np.asarray(blur_k, F32)
        k = np.broadcast_to(k32.reshape(-1, k32.shape[-1]), (box.shape[0], k32.shape[-1])).astype(ft)
    if k is not None and mutant != "blur_after_flip":
        x = blur(x, k, mutant)
    if flags & FLIP:
        x = x[..., ::-1]
    if k is not None and mutant == "blur_after_flip":
        x = blur(x, k)
    mean_n = np.array([ft(F32(v)) for v in norm[:3]], ft)[None, :, None, None]
    std_n = np.array([ft(F32(v)) for v in norm[3:]], ft)[None, :, None, None]
    return (x - mean_n) / std_n, mean
