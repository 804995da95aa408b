"""The case table of the augmentation and resize kernels (csrc/augment.cu), shared by test_host_augment_exact.py (the
oracle against torchvision and float64) and test_gpu_augment_exact.py (the kernels against the oracle).

Each AugCase is one moco_augment_crops call: one source image, one output size and a few crop records on it; each
ResizeCase one moco_resize_center_crops call of one record.  Output sizes 1x1, 1x1024, 1024x1, 7x13, 224x224,
225x257 and 1024x1024; whole images, 1x1 crops (upscaled up to 1024x), 1-pixel-wide full-height crops, crops with
about 2000 vertical taps, crops exactly 1000 * out_w wide, boxes 2048 and 2049 wide and the widths where the
column-chunk width changes, crops against the right and bottom edges (the kernels place each case's image last in the
buffer, so those read its last byte); no flags, GRAY, FLIP, JITTER and all three; all 24 jitter orders with factors
at 0.6 / 1.0 / 1.4 and hue at -0.5, 0, +-1e-7 and 0.5; and planted pixels for hue's edge cases.
"""
from __future__ import annotations

import itertools
from dataclasses import dataclass, field

import numpy as np

GRAY, FLIP, JITTER = 1, 2, 4
IDENTITY_ORDER = 0 | (1 << 2) | (2 << 4) | (3 << 6)


def order_word(perm):
    return sum(op << (2 * k) for k, op in enumerate(perm))


# (flags, jitter order, brightness, contrast, saturation, hue)
VARIANTS = [
    (0, IDENTITY_ORDER, 1.0, 1.0, 1.0, 0.0),
    (GRAY, IDENTITY_ORDER, 1.0, 1.0, 1.0, 0.0),
    (FLIP, IDENTITY_ORDER, 1.0, 1.0, 1.0, 0.0),
    (JITTER, order_word((3, 1, 0, 2)), 1.4, 0.6, 1.4, 0.5),
    (GRAY | FLIP | JITTER, order_word((2, 0, 3, 1)), 0.6, 1.4, 0.6, -0.5),
]
PLAIN, ALL3 = [VARIANTS[0]], [VARIANTS[0], VARIANTS[4]]
HUES = (-0.5, 0.0, 1e-7, -1e-7, 0.5)
FACTORS = (0.6, 1.0, 1.4)


def image(h, w, seed):
    """Smooth structure plus noise, a grey block and a white corner (test_gpu_augment's pattern), uint8 [h, w, 3]."""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (h, w, 3), dtype=np.int64)
    yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    smooth = np.stack([(yy * 255) // max(h - 1, 1), (xx * 255) // max(w - 1, 1), ((yy + xx) * 7) % 256], -1)
    img = ((base + 3 * smooth) // 4).astype(np.uint8)
    img[: h // 8, : w // 8] = 128
    img[-2:, -2:] = 255
    return img


# hue's edge cases: primaries, secondaries (h * 6 on a sector boundary), channel ties r = g > b, g = b > r, r = b > g
# and the single-maximum ties, greys, and one-level chromas
PLANTED = [(255, 0, 0), (0, 255, 0), (0, 0, 255), (255, 255, 0), (0, 255, 255), (255, 0, 255),
           (200, 200, 50), (30, 180, 180), (220, 40, 220), (200, 60, 60), (60, 200, 60), (60, 60, 200),
           (0, 0, 0), (128, 128, 128), (255, 255, 255), (101, 100, 100), (100, 101, 100), (100, 100, 101),
           (255, 254, 255), (1, 0, 0), (128, 64, 0), (0, 128, 64), (64, 0, 128)]


def planted_image(h, w, seed):
    img = image(h, w, seed)
    flat = img.reshape(-1, 3)
    flat[:len(PLANTED)] = PLANTED
    return img


@dataclass
class AugCase:
    name: str
    out: tuple                       # (out_h, out_w)
    src: tuple                       # (h, w, seed, planted)
    crops: list = field(default_factory=list)      # (top, left, height, width, flags, order, b, c, s, hue)

    def image(self):
        h, w, seed, planted = self.src
        return planted_image(h, w, seed) if planted else image(h, w, seed)


@dataclass
class ResizeCase:
    name: str
    out: tuple                       # (out_h, out_w)
    src: tuple                       # (h, w, seed)
    resized: tuple                   # (resized_h, resized_w)
    window: tuple                    # (top, left)

    def image(self):
        return image(*self.src)


def _case(name, out, src, boxes, variants):
    planted = len(src) > 3 and src[3]
    crops = [tuple(box) + tuple(v) for box in boxes for v in variants]
    return AugCase(name, out, (src[0], src[1], src[2], planted), crops)


def aug_cases():
    C = []
    # 1 x 1
    C.append(_case("1x1/whole,1px,edge", (1, 1), (300, 400, 1), [(0, 0, 300, 400), (7, 9, 1, 1), (0, 399, 300, 1),
                                                                  (295, 395, 5, 5)], VARIANTS))
    C.append(_case("1x1/tall", (1, 1), (1000, 40, 2), [(0, 5, 1000, 3)], VARIANTS))
    C.append(_case("1x1/1000x", (1, 1), (4, 1000, 3), [(1, 0, 3, 1000)], VARIANTS))
    # 1 x 1024
    C.append(_case("1x1024/1000x", (1, 1024), (2, 1024000, 4), [(0, 0, 2, 1024000)], ALL3))
    C.append(_case("1x1024/tall,2049", (1, 1024), (1000, 2049, 5), [(0, 0, 1000, 2049)], [VARIANTS[3]]))
    C.append(_case("1x1024/whole,1px", (1, 1024), (30, 40, 6), [(0, 0, 30, 40), (29, 39, 1, 1)], ALL3))
    # 1024 x 1
    C.append(_case("1024x1/whole,1px-wide", (1024, 1), (300, 400, 7), [(0, 0, 300, 400), (0, 399, 300, 1)], VARIANTS))
    C.append(_case("1024x1/1000x", (1024, 1), (40, 2049, 8), [(0, 0, 40, 1000), (3, 1049, 37, 1000)], ALL3))
    # 7 x 13
    orders = []
    for k, perm in enumerate(itertools.permutations(range(4))):
        f = [FACTORS[(k + j) % 3] for j in range(3)]
        flags = JITTER | (FLIP if k % 2 else 0) | (GRAY if k % 5 == 0 else 0)
        orders.append((flags, order_word(perm), *f, HUES[k % 5]))
    C.append(_case("7x13/24 orders", (7, 13), (181, 243, 9), [(4, 6, 170, 230)], orders))
    hue_variants = [(JITTER, order_word(p), b, c, s, hue) for hue in HUES
                    for p, (b, c, s) in [((3, 0, 1, 2), (1.0, 1.0, 1.0)), ((0, 3, 2, 1), (1.4, 0.6, 1.0)),
                                         ((2, 1, 0, 3), (1.0, 1.4, 0.6))]]
    C.append(_case("7x13/planted hue", (7, 13), (7, 13, 10, True), [(0, 0, 7, 13)], hue_variants))
    C.append(_case("7x13/1000x,1px", (7, 13), (9, 13000, 11), [(1, 0, 8, 13000), (8, 12999, 1, 1)], VARIANTS))
    # 224 x 224
    C.append(_case("224/whole,edges,1px", (224, 224), (375, 500, 12), [(0, 0, 375, 500), (200, 300, 175, 200),
                                                                         (100, 20, 1, 1)], VARIANTS))
    for ww in (2048, 2049, 2053, 2054):      # unchunked, chunked; int(2044 / sx) = 223 -> 222 between 2053 and 2054
        C.append(_case(f"224/ww={ww}", (224, 224), (300, ww, 13 + ww), [(0, 0, 300, ww)], ALL3))
    # 225 x 257: int(2044 / sx) is exactly 256 at ww = 2052 in exact arithmetic
    for ww in (2049, 2052, 2053):
        C.append(_case(f"225x257/ww={ww}", (225, 257), (333, ww, 20 + ww), [(0, 0, 333, ww)], ALL3))
    C.append(_case("225x257/edge", (225, 257), (260, 300, 21), [(10, 40, 250, 260)], VARIANTS))
    # 1024 x 1024
    C.append(_case("1024/whole", (1024, 1024), (1100, 1300, 22), [(0, 0, 1100, 1300)], ALL3))
    for ww in (2049, 2336, 2337):            # int(2044 / sx) = 896 exactly at 2336
        C.append(_case(f"1024/ww={ww}", (1024, 1024), (1030, ww, 23 + ww), [(0, 0, 1030, ww)], [VARIANTS[4]]))
    return C


def resize_cases():
    R = [ResizeCase("1x1", (1, 1), (300, 400, 31), (1, 1), (0, 0)),
         ResizeCase("7x13/1x1 up", (7, 13), (1, 1, 32), (20, 30), (13, 17)),
         ResizeCase("7x13/2x3 up", (7, 13), (2, 3, 33), (7, 13), (0, 0)),
         ResizeCase("7x13/1x2000", (7, 13), (1, 2000, 34), (7, 13), (0, 0)),
         ResizeCase("7x13/1000x", (7, 13), (5, 13000, 35), (7, 13), (0, 0)),
         ResizeCase("224/plain", (224, 224), (300, 400, 36), (256, 341), (16, 58)),
         ResizeCase("224/identity", (224, 224), (256, 300, 37), (256, 300), (16, 38)),
         ResizeCase("224/2049 wide, last left", (224, 224), (300, 2049, 38), (256, 1748), (32, 1524)),
         ResizeCase("224/4000 wide", (224, 224), (3000, 4000, 39), (256, 341), (16, 58)),
         ResizeCase("225x257/2049, last top", (225, 257), (333, 2049, 40), (260, 1600), (35, 1343)),
         ResizeCase("1024/plain", (1024, 1024), (1100, 1300, 41), (1024, 1210), (0, 186)),
         ResizeCase("1024/1x1 up", (1024, 1024), (1, 1, 42), (1024, 1024), (0, 0))]
    return R


NORM = (0.485, 0.456, 0.406, 0.229, 0.224, 0.225)


def records(case, offset=0):
    """int32 [n, 14] moco_aug_crop records of an AugCase with its image at byte ``offset``."""
    h, w = case.src[0], case.src[1]
    rows = []
    for top, left, ch, cw, flags, order, *f in case.crops:
        bits = np.array(f, np.float32).view(np.int32).tolist()
        rows.append([offset & 0xFFFFFFFF, offset >> 32, h, w, top, left, ch, cw, flags, order] + bits)
    return np.array(rows, np.int64).astype(np.uint32).view(np.int32)


def window_record(case, offset=0):
    """int32 [1, 8] moco_resize_window record of a ResizeCase with its image at byte ``offset``."""
    r = [offset & 0xFFFFFFFF, offset >> 32, case.src[0], case.src[1], *case.resized, *case.window]
    return np.array([r], np.int64).astype(np.uint32).view(np.int32)


def oracle_aug(case, img=None, exact=True, mutant=None):
    """(out [n, 3, out_h, out_w], means [n]) of an AugCase by the oracle."""
    from oracle import augment_oracle as O
    img = case.image() if img is None else img
    outs, means = [], []
    for top, left, ch, cw, flags, order, *f in case.crops:
        box = img[top:top + ch, left:left + cw][None]
        o, m = O.augment(box, *case.out, flags, order, np.array([f], np.float32), NORM, exact=exact, mutant=mutant)
        outs.append(o[0])
        means.append(m[0])
    return np.stack(outs), np.array(means)


def oracle_resize(case, img=None, exact=True, mutant=None):
    from oracle import augment_oracle as O
    img = case.image() if img is None else img
    return O.resize_window(img[None], *case.resized, *case.window, *case.out, NORM, exact=exact, mutant=mutant)
