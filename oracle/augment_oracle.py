"""An exact numpy restatement of moco_augment_crops and moco_resize_center_crops (include/moco_b200.h,
moco_b200/csrc/augment.cu), written from the header contract and the kernel's documented operation order.

It shares no code with the kernels or with moco_b200/augment.py's host code; only the record word indices and the
flag bits are the same numbers.  One call evaluates a batch of crops that share one geometry (source box, output size,
flags and jitter order; the factors may differ per crop), on the whole crop at once: no column chunks, no row tiles,
no threads.  The chunk width is computed only where the contract's summation order depends on it, the contrast mean.

Two modes:
  * ``exact=True``: every operation is one numpy float32 operation, rounded to nearest, in the kernel's order:
      - tap geometry (ATen's upsample_bilinear2d_aa): scale = f32(in) / f32(out), center = f32(double(scale) * (i +
        0.5)), the tap range [lo, lo + n) in double, invscale = f32(1 / double(scale)); weight = (1 - |((k - center) +
        0.5) * invscale|) * f32(1 / total), total the tap-order sum of the unnormalised weights;
      - the vertical pass on raw uint8 values, summed in tap order, then / 255; the horizontal pass in tap order;
      - gray, _blend with fm = f32(1 - double(f)), the hue round trip (fmod, remainder, floor, i % 6) as written;
      - the contrast mean: thread t of 256 sums columns a + t, a + t + 256, ... of each column chunk [a, a + cw) of
        each row (rows outermost), the lanes are folded by v += v[lane ^ s] for s = 16 ... 1, warps 0 ... 7 are added
        in order and the total is divided once by f32(out_h * out_w);
      - the flip, then (x - mean) / std.
    The result is what the kernels must return bit for bit.
  * ``exact=False``: the high-precision reference.  The same geometry (float32 scale, center and invscale, tap
    ranges) and the same float32-rounded constants (factors, gray weights, mean and std), with every other operation
    in float64.

``mutant`` names a deliberately wrong variant (MUTANTS); the tests use them to show that a case table catches such
errors.  None is the contract.
"""
from __future__ import annotations

import numpy as np

F32, F64 = np.float32, np.float64
SPAN = 2048                       # source pixels one column chunk may span
THREADS, WARP = 256, 32           # the contrast-mean CTA
GRAY, FLIP, JITTER = 1, 2, 4      # record flag bits
GRAY_W = (F32(0.2989), F32(0.587), F32(0.114))

MUTANTS = ("drop_last_vtap", "drop_last_htap", "div255_first", "mean_skip_last_row", "mean_skip_last_chunk",
           "chunk2_x0_plus_1", "flip_out_w_minus_sx")
SEMANTIC_MUTANTS = tuple(m for m in MUTANTS if m != "div255_first")    # the rest only change rounding


class Taps:
    """The taps of output indices ``idx`` of a resample of ``in_size`` source pixels to ``out_size``.
    lo, n: int64 [len(idx)]; w32 / w64: float32 / float64 [len(idx), max_n] weights, zero past tap n - 1;
    total: float64 [len(idx)], the sum of the unnormalised float64 weights."""

    def __init__(self, idx, in_size, out_size):
        scale = F32(F32(in_size) / F32(out_size))
        support = scale if scale >= 1 else F32(1)
        invscale = F32(1.0 / F64(scale)) if scale >= 1 else F32(1)
        i = np.asarray(idx, np.int64)
        center = (F64(scale) * (i.astype(F64) + 0.5)).astype(F32)
        self.max_n = max_n = int(np.ceil(F64(support))) * 2 + 1
        lo = np.maximum(((center - support).astype(F64) + 0.5).astype(np.int64), 0)
        hi = np.minimum(((center + support).astype(F64) + 0.5).astype(np.int64), in_size)
        n = np.maximum(0, np.minimum(hi - lo, max_n))
        k = lo[:, None] + np.arange(max_n)
        valid = np.arange(max_n) < n[:, None]
        x32 = np.abs(((k.astype(F32) - center[:, None]) + F32(0.5)) * invscale)
        t32 = np.where(valid & (x32 < 1), F32(1) - x32, F32(0)).astype(F32)
        total32 = np.zeros(len(i), F32)
        for j in range(max_n):                                   # tap order
            total32 = total32 + t32[:, j]
        norm = np.where(total32 != 0, (1.0 / np.where(total32 != 0, total32, 1).astype(F64)).astype(F32), F32(0))
        self.w32 = np.where(t32 != 0, t32 * norm[:, None], F32(0)).astype(F32)
        x64 = np.abs((k.astype(F64) - center[:, None].astype(F64) + 0.5) * F64(invscale))
        t64 = np.where(valid & (x64 < 1), 1.0 - x64, 0.0)
        self.total = t64.sum(axis=1)
        self.w64 = t64 / np.where(self.total != 0, self.total, 1)[:, None]
        self.lo, self.n, self.scale = lo, n, scale

    def drop_last(self):
        last = (self.n - 1)[:, None] == np.arange(self.max_n)
        self.w32 = np.where(last, F32(0), self.w32)
        self.w64 = np.where(last, 0.0, self.w64)


def chunk_width(ww, dst_w, out_w):
    """Output columns per column chunk, as the kernel computes it: out_w when the box is at most SPAN pixels wide,
    else max(1, min(out_w, int(f32(SPAN - 4) / f32 scale) - 1))."""
    if ww <= SPAN:
        return out_w
    sx = F32(F32(ww) / F32(dst_w))
    return max(1, min(out_w, int(F32(SPAN - 4) / sx) - 1))


def _resample(box, ty, tx, exact, mutant, cw):
    """box: uint8 [N, hh, ww, 3] -> [N, len(ty), len(tx), 3]: the vertical pass on raw values in tap order, / 255,
    then the horizontal pass in tap order."""
    ft = F32 if exact else F64
    wy, wx = (ty.w32, tx.w32) if exact else (ty.w64, tx.w64)
    hh, ww = box.shape[1], box.shape[2]
    acc = np.zeros((box.shape[0], len(ty.lo), ww, 3), ft)
    for j in range(ty.max_n):
        rows = np.minimum(ty.lo + j, hh - 1)
        px = box[:, rows].astype(ft)
        if mutant == "div255_first":
            px = px / ft(255)
        acc = acc + wy[None, :, j, None, None] * px
    v = acc if mutant == "div255_first" else acc / ft(255)
    shift = np.zeros(len(tx.lo), bool)
    if mutant == "chunk2_x0_plus_1" and cw < len(tx.lo):
        # chunk [cw, 2 cw) loads its span from one column too far right; a tap left of it clamps onto its first column
        shift[cw:2 * cw] = True
    out = np.zeros((box.shape[0], len(ty.lo), len(tx.lo), 3), ft)
    for j in range(tx.max_n):
        cols = tx.lo + j
        if shift.any():
            cols = np.where(shift, np.maximum(cols, tx.lo[cw] + 1), cols)
        out = out + wx[None, None, :, j, None] * v[:, :, np.minimum(cols, ww - 1)]
    return out[..., 0], out[..., 1], out[..., 2]


def gray(r, g, b):
    ft = r.dtype.type
    return (ft(GRAY_W[0]) * r + ft(GRAY_W[1]) * g) + ft(GRAY_W[2]) * b


def _blend(a, b, f, fm):
    return np.minimum(np.maximum(f * a + fm * b, 0), 1).astype(a.dtype)


def hue_shift(r, g, b, hue):
    """torchvision's _rgb2hsv, h = (h + hue) % 1.0 (torch.remainder), _hsv2rgb, in the kernel's order."""
    ft = r.dtype.type
    one = ft(1)
    maxc = np.maximum(r, np.maximum(g, b))
    minc = np.minimum(r, np.minimum(g, b))
    eqc = maxc == minc
    cr = maxc - minc
    s = cr / np.where(eqc, one, maxc)
    crd = np.where(eqc, one, cr)
    rc, gc, bc = (maxc - r) / crd, (maxc - g) / crd, (maxc - b) / crd
    hr = np.where(maxc == r, bc - gc, ft(0))
    hg = np.where((maxc == g) & (maxc != r), (ft(2) + rc) - bc, ft(0))
    hb = np.where((maxc != g) & (maxc != r), (ft(4) + gc) - rc, ft(0))
    h = np.fmod(((hr + hg) + hb) / ft(6) + one, one)
    h = np.fmod(h + hue, one)
    h = np.where(h < 0, h + one, h)
    h6 = h * ft(6)
    fi = np.floor(h6)
    f = h6 - fi
    i = np.mod(fi.astype(np.int64), 6)
    v = maxc
    p = np.minimum(np.maximum(v * (one - s), 0), 1)
    q = np.minimum(np.maximum(v * (one - s * f), 0), 1)
    t = np.minimum(np.maximum(v * (one - s * (one - f)), 0), 1)
    sel = [i == k for k in range(6)]
    r2 = np.select(sel, [v, q, p, p, t, v])
    g2 = np.select(sel, [t, v, v, q, p, p])
    b2 = np.select(sel, [p, p, t, v, v, q])
    return r2.astype(ft), g2.astype(ft), b2.astype(ft)


def _pointwise(r, g, b, flags, order, factors, mean):
    """The ops after the resample; with mean None, stop before the contrast op and return its input."""
    ft = r.dtype.type
    if flags & GRAY:
        r = g = b = gray(r, g, b)
    if not flags & JITTER:
        return r, g, b
    f = factors.astype(ft)[:, :, None, None]                     # [N, 4, 1, 1]
    fm = (1.0 - factors.astype(F64)).astype(F32).astype(ft)[:, :, None, None]
    for k in range(4):
        op = (order >> (2 * k)) & 3
        fk, fmk = f[:, op], fm[:, op]
        if op == 0:
            zero = np.zeros_like(r)
            r, g, b = (_blend(x, zero, fk, fmk) for x in (r, g, b))
        elif op == 1:
            if mean is None:
                return r, g, b
            m = mean.astype(ft)[:, None, None]
            r, g, b = (_blend(x, m, fk, fmk) for x in (r, g, b))
        elif op == 2:
            lum = gray(r, g, b)
            r, g, b = (_blend(x, lum, fk, fmk) for x in (r, g, b))
        else:
            r, g, b = hue_shift(r, g, b, fk)
    return r, g, b


def thread_columns(out_w, cw, mutant=None):
    """[THREADS] lists of the columns thread t adds within one output row, in its order."""
    starts = list(range(0, out_w, cw))
    if mutant == "mean_skip_last_chunk":
        starts = starts[:-1]
    return [np.concatenate([np.arange(a + t, min(a + cw, out_w), THREADS) for a in starts] + [np.zeros(0, np.int64)])
            for t in range(THREADS)]


def contrast_mean(lum, cw, mutant=None):
    """The fixed-order float32 mean of lum [N, out_h, out_w] (the crops' pre-contrast grayscale) with column chunks
    of cw: per-thread sequential sums (rows outermost), the xor-shuffle fold, then warps 0 ... 7 in order."""
    n, out_h, out_w = lum.shape
    cols = thread_columns(out_w, cw, mutant)
    width = max(len(c) for c in cols)
    idx = np.zeros((THREADS, width), np.int64)
    live = np.zeros((THREADS, width), bool)
    for t, c in enumerate(cols):
        idx[t, :len(c)], live[t, :len(c)] = c, True
    rows = out_h - 1 if mutant == "mean_skip_last_row" else out_h
    acc = np.zeros((n, THREADS), F32)
    for oy in range(rows):
        row = lum[:, oy]
        for m in range(width):
            acc = acc + np.where(live[:, m], row[:, idx[:, m]], F32(0))      # + 0 leaves a sum >= 0 unchanged
    lanes = acc.reshape(n, THREADS // WARP, WARP)
    for s in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, :, np.arange(WARP) ^ s]
    total = np.zeros(n, F32)
    for w in range(THREADS // WARP):
        total = total + lanes[:, w, 0]
    return total / F32(out_h * out_w)


def _normalize(r, g, b, flags, norm, mutant):
    ft = r.dtype.type
    x = np.stack([r, g, b], axis=1)                              # [N, 3, H, W]
    if flags & FLIP:
        if mutant == "flip_out_w_minus_sx":
            w = x.shape[-1]
            x = x[..., (w - np.arange(w)) % w]
        else:
            x = x[..., ::-1]
    mean = np.array([ft(F32(v)) for v in norm[:3]], ft)[None, :, None, None]
    std = np.array([ft(F32(v)) for v in norm[3:]], ft)[None, :, None, None]
    return (x - mean) / std


def augment(box, out_h, out_w, flags, order, factors, norm, exact=True, mutant=None):
    """moco_augment_crops on N crops of one geometry.  box: uint8 [N, hh, ww, 3], each crop's box cut from its image;
    factors: float32 [N, 4] (brightness, contrast, saturation, hue).  Returns (out [N, 3, out_h, out_w], crop means
    [N], 0 where jitter is off), float32 when exact else float64."""
    box = np.asarray(box, np.uint8)
    factors = np.asarray(factors, F32).reshape(-1, 4)
    hh, ww = box.shape[1], box.shape[2]
    ty, tx = Taps(np.arange(out_h), hh, out_h), Taps(np.arange(out_w), ww, out_w)
    if mutant == "drop_last_vtap":
        ty.drop_last()
    if mutant == "drop_last_htap":
        tx.drop_last()
    cw = chunk_width(ww, out_w, out_w)
    r, g, b = _resample(box, ty, tx, exact, mutant, cw)
    ft = F32 if exact else F64
    mean = np.zeros(box.shape[0], ft)
    if flags & JITTER:
        lum = gray(*_pointwise(r, g, b, flags, order, factors, None))
        if exact:
            mean = contrast_mean(lum, cw, mutant)
        else:
            mean = lum.mean(axis=(1, 2))
    r, g, b = _pointwise(r, g, b, flags, order, factors, mean)
    return _normalize(r, g, b, flags, norm, mutant), mean


def resize_window(src, resized_h, resized_w, top, left, out_h, out_w, norm, exact=True, mutant=None):
    """moco_resize_center_crops on N sources of one size: uint8 [N, src_h, src_w, 3] resampled whole to resized_h x
    resized_w, of which rows [top, top + out_h) and columns [left, left + out_w) are evaluated (the window's origin
    on the tap index).  Returns [N, 3, out_h, out_w]."""
    src = np.asarray(src, np.uint8)
    ty = Taps(top + np.arange(out_h), src.shape[1], resized_h)
    tx = Taps(left + np.arange(out_w), src.shape[2], resized_w)
    if mutant == "drop_last_vtap":
        ty.drop_last()
    if mutant == "drop_last_htap":
        tx.drop_last()
    cw = chunk_width(src.shape[2], resized_w, out_w)
    r, g, b = _resample(src, ty, tx, exact, mutant, cw)
    return _normalize(r, g, b, 0, norm, mutant)
