"""The case table of moco_augment_crops_blur (MoCo v2's records, csrc/augment.cu), shared by test_host_augment_v2.py
(the oracle against torchvision and float64, the blur mutants) and test_gpu_augment_v2.py (the kernels against the
oracle, bit for bit).

Each BlurCase is one call: one source image, one output size, one ksize and a few 32-word records on it, blurred and
unblurred crops mixed in the same batch.  ksize 3, 23 and 31; sigma 0.1 (the outer taps underflow to 0) and 2.0;
16 x 16 with ksize 31, where the reflect halo reaches the far edge; output heights that are not a multiple of the blur
pass's band (37, 100, 225) and a 512-wide output where the band is 2 rows; flip on and off; grayscale after the
jitter with the jitter applied and not applied, and the v1 order on a blurred crop.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from moco_b200.augment import gaussian_half_kernel
from tests import augment_cases as AC

GRAY, FLIP, JITTER = AC.GRAY, AC.FLIP, AC.JITTER
ID = AC.IDENTITY_ORDER
NORM = AC.NORM

# (flags, jitter order, brightness, contrast, saturation, hue, gray_after_jitter, blur, sigma)
VARIANTS = [
    (0, ID, 1.0, 1.0, 1.0, 0.0, 1, 1, 2.0),                                       # blur alone
    (FLIP, ID, 1.0, 1.0, 1.0, 0.0, 1, 1, 0.1),                                    # sigma 0.1, flipped
    (JITTER | GRAY, AC.order_word((3, 1, 0, 2)), 1.4, 0.6, 1.4, 0.1, 1, 1, 2.0),  # gray after the jitter, blurred
    (GRAY | FLIP, ID, 1.0, 1.0, 1.0, 0.0, 1, 0, None),                            # gray after a jitter not applied
    (JITTER | GRAY | FLIP, AC.order_word((2, 0, 3, 1)), 0.6, 1.4, 0.6, -0.1, 1, 0, None),
    (JITTER | GRAY | FLIP, AC.order_word((0, 2, 1, 3)), 1.2, 0.8, 0.7, 0.05, 0, 1, 1.3),   # v1 order, blurred
    (0, ID, 1.0, 1.0, 1.0, 0.0, 0, 0, None),                                      # plain
]


@dataclass
class BlurCase:
    name: str
    out: tuple                       # (out_h, out_w)
    src: tuple                       # (h, w, seed)
    ksize: int
    crops: list = field(default_factory=list)      # (top, left, height, width) + a VARIANTS entry

    def image(self):
        return AC.image(*self.src)


def _case(name, out, src, ksize, boxes, variants=VARIANTS):
    return BlurCase(name, out, src, ksize, [tuple(b) + tuple(v) for b in boxes for v in variants])


def cases():
    return [
        _case("224/k23", (224, 224), (375, 500, 60), 23, [(0, 0, 375, 500), (200, 300, 175, 200)]),
        _case("224/k3", (224, 224), (300, 260, 61), 3, [(10, 20, 280, 230)], VARIANTS[:3] + VARIANTS[5:]),
        _case("16/k31", (16, 16), (40, 50, 62), 31, [(0, 0, 40, 50), (5, 7, 3, 4)]),
        _case("37x41/k23", (37, 41), (90, 120, 63), 23, [(3, 4, 80, 110)]),
        _case("100x60/k31", (100, 60), (150, 130, 64), 31, [(0, 0, 150, 130)], VARIANTS[:3]),
        _case("225x97/k23", (225, 97), (250, 300, 65), 23, [(0, 10, 240, 290)], VARIANTS[1:3] + VARIANTS[6:]),
        _case("512/k31", (512, 512), (600, 700, 66), 31, [(0, 0, 600, 700)], VARIANTS[2:4]),
    ]


def kernel1d(ksize, sigma):
    """The full 1-D kernel of torchvision's _get_gaussian_kernel1d(ksize, sigma, float32), via the host's weights."""
    half = np.array(gaussian_half_kernel(ksize, sigma), np.float32)[:ksize // 2 + 1]
    return np.concatenate([half[:0:-1], half])


def records(case, offset=0):
    """int32 [n, 32] moco_aug_crop_blur records of a BlurCase with its image at byte ``offset``."""
    h, w = case.src[0], case.src[1]
    rows = []
    for top, left, ch, cw, flags, order, b, c, s, hue, late, blur, sigma in case.crops:
        wts = gaussian_half_kernel(case.ksize, sigma) if blur else [0.0] * 16
        bits = np.array([b, c, s, hue], np.float32).view(np.int32).tolist()
        rows.append([offset & 0xFFFFFFFF, offset >> 32, h, w, top, left, ch, cw, flags, order] + bits +
                    [late, blur] + np.array(wts, np.float32).view(np.int32).tolist())
    return np.array(rows, np.int64).astype(np.uint32).view(np.int32)


def oracle(case, img=None, exact=True, mutant=None):
    """(out [n, 3, out_h, out_w], means [n]) of a BlurCase by the oracle (tests/augment_blur_oracle.py)."""
    from tests import augment_blur_oracle as BO
    img = case.image() if img is None else img
    outs, means = [], []
    for top, left, ch, cw, flags, order, b, c, s, hue, late, blur, sigma in case.crops:
        box = img[top:top + ch, left:left + cw][None]
        k = kernel1d(case.ksize, sigma) if blur else None
        o, m = BO.augment(box, *case.out, flags, order, np.array([[b, c, s, hue]], np.float32), NORM, exact=exact,
                          mutant=mutant, gray_late=bool(late), blur_k=k)
        outs.append(o[0])
        means.append(m[0])
    return np.stack(outs), np.array(means)
