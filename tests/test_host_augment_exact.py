"""The exact restatement of the augmentation and resize kernels (oracle/augment_oracle.py), no GPU needed: known
values of its tap geometry, chunk width, hue round trip and contrast-mean order checked by hand; the whole case table
(tests/augment_cases.py) against torchvision's fp32 tensor ops and within a derived bound of the float64 mode; and
deliberately wrong variants of the oracle, each caught by the table (the semantic ones by the float64 bound too).

The float64 bound (``_aug_bounds`` / ``_resize_bound``), in [0, 1] units per stage then normalised; u = 2^-24, gamma_n = n u / (1 - n u).
The float64 mode shares the float32 geometry and constants, so only float32 rounding separates the two; its own
rounding (2^-53 relative) is far below the slack of the constants.
  * Weights of one output index with n taps and float64 unnormalised sum T.  Each |x| = |((k - c) + 0.5) * inv| is
    off by at most 3.5 u (|k - c| <= S + 0.5, inv = 1 / S), so each 1 - x by <= 5 u (exact when x >= 0.5, and a tap
    that switches sides of x < 1 is worth < 4 u).  Their float32 sum has relative error <= 5 n u / T + gamma_{n-1},
    the reciprocal and the product add 2 u, so sum_j |w32_j - w_j| <= E_w = 1.01 (10 n / T + n + 1) u.
  * One pass y = sum_j w_j p_j, 0 <= p_j <= P, over inputs off by e_p: the products and n - 1 additions give
    gamma_n sum_j w32_j p_j, so |y32 - y| <= P (E_w + gamma_n (1 + E_w)) + (1 + E_w) e_p.  Vertical: P = 255, e_p = 0,
    then / 255 adds 1.01 u; horizontal: P = 1 + e_v.  The resample is within e_res = (n_y + n_x + c) u.
  * Values stay in [0, A], A = 1.01.  gray: 3 products and 2 additions, e + 3 u A.  _blend(a, b, f), fm exact:
    f e_a + |fm| e_b + 2 u A (f + |fm|).  hue: the round trip is piecewise linear and continuous, each output one of
    max, min, max - cr f, min + cr f with cr f = L(rgb) + K cr, |K| <= 2, L a channel difference: Lipschitz 7.  Its
    float32 evaluation at fixed inputs: rc, gc, bc <= 3.01 u, the hue numerator <= 16.02 u, h <= 8 u, h * 6 <= 54 u,
    then p, q, t <= 61 u: 7 e + 64 u.
  * The contrast mean: each term passes at most L + 11 roundings (L terms per thread, 5 shuffle and 7 warp
    additions), so it is off by e_gray + 1.01 (L + 12) u A.  Brightness blends with an exact 0.
  * Normalize: (e + u) / std * 1.001 + 3 u.
"""
import itertools

import numpy as np
import pytest
import torch
from torchvision.transforms import functional as TF

from oracle import augment_oracle as O
from tests import augment_cases as AC

U = 2.0 ** -24
A = 1.01
TORCHVISION_MEASURED = 1.12e-5         # max |oracle - torchvision fp32| over the table, normalised units (7x13 from
TORCHVISION_BOUND = 2e-5               # a 13000-wide crop: 2000-tap sums in another order)


def _tv_aug(img, case, k):
    from moco_b200 import augment as MA
    rec = torch.from_numpy(AC.records(case)[k].copy())
    return MA.reference_crop(torch.from_numpy(img), rec, case.out).numpy()


def _tv_resize(img, case):
    x = torch.from_numpy(img).permute(2, 0, 1).float() / 255
    x = TF.resize(x, list(case.resized), antialias=True)
    (t, l), (h, w) = case.window, case.out
    return TF.normalize(x[:, t:t + h, l:l + w], list(AC.NORM[:3]), list(AC.NORM[3:])).numpy()


# ------------------------------------------------------------------------------------------------ the float64 bound

def _gamma(n):
    return n * U / (1 - n * U)


def _pass_bound(taps, P, e_p):
    n, T = taps.n.astype(float), taps.total
    ew = 1.01 * (10 * n / np.maximum(T, 1e-300) + n + 1) * U
    return float(np.max(P * (ew + _gamma(n) * (1 + ew)) + (1 + ew) * e_p))


def _resample_bound(ty, tx):
    e_v = _pass_bound(ty, 255.0, 0.0) / 255.0 + 1.01 * U
    return _pass_bound(tx, 1.0 + e_v, e_v)


def _blend_err(f, fm, e_a, e_b):
    return f * e_a + abs(fm) * e_b + 2 * U * A * (f + abs(fm))


def _pointwise_bound(e, flags, order, factors, L):
    """Error after the ops given the resample's e; the contrast mean's from the same path to the contrast op."""
    if flags & AC.GRAY:
        e = e + 3 * U * A
    if not flags & AC.JITTER:
        return e
    f = [float(np.float32(v)) for v in factors]
    fm = [float(np.float32(1.0 - v)) for v in f]
    for k in range(4):
        op = (order >> (2 * k)) & 3
        if op == 0:
            e = _blend_err(f[0], fm[0], e, 0.0)
        elif op == 1:
            e_m = e + 3 * U * A + 1.01 * (L + 12) * U * A
            e = _blend_err(f[1], fm[1], e, e_m)
        elif op == 2:
            e = _blend_err(f[2], fm[2], e, e + 3 * U * A)
        else:
            e = 7 * e + 64 * U
    return e


def _normalized(e):
    return (e + U) / min(AC.NORM[3:]) * 1.001 + 3 * U


def _terms_per_thread(out_h, out_w, cw):
    return out_h * max(len(c) for c in O.thread_columns(out_w, cw))


def _aug_bounds(case):
    out_h, out_w = case.out
    bounds = []
    for top, left, ch, cw, flags, order, *f in case.crops:
        ty, tx = O.Taps(np.arange(out_h), ch, out_h), O.Taps(np.arange(out_w), cw, out_w)
        L = _terms_per_thread(out_h, out_w, O.chunk_width(cw, out_w, out_w))
        bounds.append(_normalized(_pointwise_bound(_resample_bound(ty, tx), flags, order, f, L)))
    return np.array(bounds)


def _resize_bound(case):
    (rh, rw), (t, l), (oh, ow) = case.resized, case.window, case.out
    ty = O.Taps(t + np.arange(oh), case.src[0], rh)
    tx = O.Taps(l + np.arange(ow), case.src[1], rw)
    return _normalized(_resample_bound(ty, tx))


# ------------------------------------------------------------------------------------------------------ by hand

def test_tap_geometry_by_hand():
    # scale 1: one tap of weight 1 and a zero tap beside it
    t = O.Taps(np.arange(5), 5, 5)
    assert t.lo.tolist() == [0, 1, 2, 3, 4] and t.n.tolist() == [2, 2, 2, 2, 1]
    assert t.w32[:, 0].tolist() == [1.0] * 5 and t.w32[:4, 1].tolist() == [0.0] * 4
    # scale 1/224 (a 1-pixel box upscaled): one tap, weight t * f32(1 / t) with t = 1 - |(0 - c) + 0.5|
    t = O.Taps(np.arange(224), 1, 224)
    assert t.lo.tolist() == [0] * 224 and t.n.tolist() == [1] * 224
    s = np.float32(1) / np.float32(224)
    for i in (0, 111, 223):
        c = np.float32(float(s) * (i + 0.5))
        tri = np.float32(1) - np.abs((np.float32(0) - c) + np.float32(0.5))
        assert t.w32[i, 0] == tri * np.float32(1.0 / float(tri))
    # scale 2049 / 1024 = 2.0009765625 exactly: output 0 has center 1.00048828125, taps [0, 3) of at most 7
    t = O.Taps(np.arange(1024), 2049, 1024)
    assert t.max_n == 7 and (t.lo[0], t.n[0]) == (0, 3)
    assert (t.lo[1], t.n[1]) == (1, 4)                     # c = 3.00146484375: [int(1.5005), int(5.5024))
    # scale 1000: 1000 taps of 2001, symmetric about the center 500, summing to 1 within a few ulps
    t = O.Taps(np.arange(1), 1000, 1)
    assert t.max_n == 2001 and (t.lo[0], t.n[0]) == (0, 1000)
    w = t.w32[0, :1000]
    assert np.array_equal(w, w[::-1]) and w[499] == w.max()
    assert abs(float(w.astype(np.float64).sum()) - 1.0) < 1e-5


def test_chunk_width_by_hand():
    assert O.chunk_width(2048, 224, 224) == 224 and O.chunk_width(2048, 1024, 1024) == 1024
    assert O.chunk_width(2049, 224, 224) == 222            # 2044 / 9.1473 = 223.45
    assert O.chunk_width(2049, 1024, 1024) == 1020         # 2044 / 2.0009765625 = 1021.5
    assert O.chunk_width(2053, 224, 224) == 222 and O.chunk_width(2054, 224, 224) == 221
    assert O.chunk_width(2336, 1024, 1024) == 895          # 2044 / 2.28125 = 896 exactly
    assert O.chunk_width(2337, 1024, 1024) == 894
    assert O.chunk_width(1024000, 1024, 1024) == 1         # 1000x: one column per chunk
    assert O.chunk_width(2049, 1, 1) == 1


def _hue(rgb, hue):
    x = np.array(rgb, np.float32).reshape(3, 1, 1, 1) / np.float32(255)
    r, g, b = O.hue_shift(x[0], x[1], x[2], np.float32(hue))
    return np.array([r.item(), g.item(), b.item()], np.float32)


def test_hue_round_trip_by_hand():
    one, zero = np.float32(1), np.float32(0)
    assert _hue((255, 0, 0), 0.0).tolist() == [one, zero, zero]
    assert _hue((255, 0, 0), np.float32(1 / 3)).tolist() == [zero, one, zero]          # h * 6 = 2 exactly
    assert _hue((255, 0, 0), -0.5).tolist() == [zero, one, one]                        # -0.5 -> 0.5: cyan
    y = _hue((0, 0, 255), 0.5)                                  # f32(2/3) + 1/2 lands just past h * 6 = 1: yellow
    assert y[1] == one and y[2] == zero and 1 - 1e-6 < y[0] < 1
    r = _hue((255, 0, 0), -1e-7)                       # h = 1 - 1e-7: sector 5, f just below 1
    assert r[0] == one and r[1] == zero and 0 < r[2] < 1e-6
    for grey in (0, 128, 255):                         # no chroma: any shift is the identity
        for h in AC.HUES:
            assert _hue((grey, grey, grey), h).tolist() == [np.float32(grey) / np.float32(255)] * 3
    # ties: r = g > b resolves to max = r, g = b > r and r = b > g likewise; a zero shift returns the input to an ulp
    for rgb in ((200, 200, 50), (30, 180, 180), (220, 40, 220), (255, 255, 0), (0, 255, 255), (255, 0, 255)):
        x = np.array(rgb, np.float32) / np.float32(255)
        assert np.abs(_hue(rgb, 0.0) - x).max() <= 2 ** -22, rgb
    # and every planted pixel at every hue is torchvision's adjust_hue bit for bit
    px = np.array(AC.PLANTED, np.float32) / np.float32(255)
    for h in AC.HUES:
        got = np.stack(O.hue_shift(px[:, 0], px[:, 1], px[:, 2], np.float32(h)), 1)
        ref = TF.adjust_hue(torch.from_numpy(px.T.copy()).view(3, -1, 1), h).view(3, -1).T.numpy()
        assert np.array_equal(got, ref), h


def test_contrast_mean_order_by_hand():
    """8 x 300, one chunk: thread 0 adds columns 0 and 256 of each row, rows outermost; thread 1 column 1; thread 32
    (warp 1) column 32."""
    lum = np.zeros((1, 8, 300), np.float32)
    lum[0, :, 256] = 2.0 ** -24
    lum[0, 7, 0] = 1.0                 # rows outermost: 7 * 2^-24 first, 1 + 3.5 ulp -> 1 + 4 ulp, then a tie to even
    lum[0, 0, 1] = 2.0 ** -23          # lane 1 joins lane 0 at the last fold step
    lum[0, 1, 32] = 0.5                # warp 1
    t0 = np.float32(1 + 2.0 ** -21)
    want = (t0 + np.float32(2.0 ** -23) + np.float32(0.5)) / np.float32(2400)
    assert O.contrast_mean(lum, 300)[0] == np.float32(want)
    # columns outermost would have absorbed every 2^-24 into 1.0
    assert np.float32(want) != (np.float32(1 + 2.0 ** -23) + np.float32(0.5)) / np.float32(2400)
    # two chunks of 150: thread 0 now adds columns 0 and 150; column 256 belongs to thread 106
    assert O.contrast_mean(lum, 150)[0] == (np.float32(1.0) + np.float32(2.0 ** -23) + np.float32(0.5) +
                                             np.float32(8 * 2.0 ** -24)) / np.float32(2400)


# ---------------------------------------------------------------------------------------------- the whole table

def test_table_is_inside_the_contract():
    """Every record passes the host validation, the 1000x downscale limit included: outside it the kernels' values
    are unspecified (one column's taps may span more source pixels than a chunk holds)."""
    from moco_b200 import augment as MA
    for case in AC.aug_cases():
        h, w = case.src[0], case.src[1]
        MA.validate_params(torch.from_numpy(AC.records(case)), h * w * 3, case.out[1])
    for case in AC.resize_cases():
        MA.validate_windows(torch.from_numpy(AC.window_record(case)), case.src[0] * case.src[1] * 3, *case.out)


@pytest.fixture(scope="module")
def table():
    """Every case with its image, fp32 oracle output and float64 output."""
    rows = []
    for case in AC.aug_cases():
        img = case.image()
        rows.append((case, img, AC.oracle_aug(case, img), AC.oracle_aug(case, img, exact=False)))
    for case in AC.resize_cases():
        img = case.image()
        rows.append((case, img, AC.oracle_resize(case, img), AC.oracle_resize(case, img, exact=False)))
    return rows


def test_table_against_torchvision(table):
    """Outputs one column wide are left to the float64 bound: there torch's CPU upsample_bilinear2d_aa returns source
    row 0 for every output row."""
    worst = 0.0
    for case, img, got, _ in table:
        if case.out[1] == 1:
            continue
        if isinstance(case, AC.AugCase):
            for k in range(len(case.crops)):
                worst = max(worst, float(np.abs(got[0][k] - _tv_aug(img, case, k)).max()))
        else:
            worst = max(worst, float(np.abs(got[0] - _tv_resize(img, case)).max()))
    print(f"max |oracle - torchvision| = {worst:.3g}")
    assert worst <= TORCHVISION_BOUND, worst


def test_table_within_the_float64_bound(table):
    tightest = 0.0
    for case, img, got, ref in table:
        if isinstance(case, AC.AugCase):
            bound = _aug_bounds(case)
            err = np.abs(got[0] - ref[0]).reshape(len(case.crops), -1).max(axis=1)
        else:
            bound, err = np.array([_resize_bound(case)]), np.array([np.abs(got[0] - ref[0]).max()])
        assert (err <= bound).all(), (case.name, err, bound)
        tightest = max(tightest, float((err / bound).max()))
    print(f"largest error / bound = {tightest:.3g}")


@pytest.mark.parametrize("mutant", O.MUTANTS)
def test_mutants_are_caught(table, mutant):
    differs = breaks = None
    for case, img, got, ref in table:
        if isinstance(case, AC.AugCase):
            mut = AC.oracle_aug(case, img, mutant=mutant)
            bound = _aug_bounds(case)[:, None]
            over = (np.abs(mut[0] - ref[0]).reshape(len(case.crops), -1) > bound).any()
            diff = not (np.array_equal(mut[0], got[0]) and np.array_equal(mut[1], got[1]))
        else:
            mut = AC.oracle_resize(case, img, mutant=mutant)
            over = (np.abs(mut - ref) > _resize_bound(case)).any()
            diff = not np.array_equal(mut, got)
        differs = differs or (case.name if diff else None)
        breaks = breaks or (case.name if over else None)
        if differs and (breaks or mutant not in O.SEMANTIC_MUTANTS):
            break
    print(f"{mutant}: differs on {differs}, breaks the float64 bound on {breaks}")
    assert differs
    if mutant in O.SEMANTIC_MUTANTS:
        assert breaks
