"""moco_augment_crops and moco_resize_center_crops (csrc/augment.cu) against their exact restatement
(oracle/augment_oracle.py), bit for bit, over the case table of tests/augment_cases.py, a 65535-crop batch (the grid
limit), a 512-crop batch drawn by the sampler and one image past byte 2^32.

The C entries are called through ctypes so that the test owns the placement of the images (each case's image starts
at an odd byte and ends at pixels_bytes) and crop_means.  fp32 outputs must be equal by value, crop_means equal for
jitter crops and 0 for the others, bf16 outputs the rounded fp32 outputs, and each call must make exactly its 2
(augment) or 1 (resize) launches.
"""
import ctypes
import itertools
import time

import numpy as np
import pytest
import torch

from moco_b200 import _lib
from moco_b200 import augment as MA
from oracle import augment_oracle as O
from tests import augment_cases as AC

pytestmark = pytest.mark.gpu
GAP = 7                              # bytes before the first image: images start unaligned
BIG_OFFSET = (1 << 32) + 3           # the image placed past 2^32
MAX_DEVICE_BYTES = 10 * 10 ** 9


def _norm():
    return (ctypes.c_float * 6)(*AC.NORM)


def _pack(images, gap=GAP):
    """uint8 device buffer holding ``images`` back to back after ``gap`` bytes, the last ending at its end; and
    each image's byte offset."""
    offsets = np.cumsum([gap] + [im.nbytes for im in images])
    host = np.zeros(int(offsets[-1]), np.uint8)
    for im, off in zip(images, offsets[:-1]):
        host[off:off + im.nbytes] = im.reshape(-1)
    return torch.from_numpy(host).cuda(), [int(o) for o in offsets[:-1]]


def _augment(pix, recs, out, dtype=torch.float32):
    """One moco_augment_crops call: (dst [n, 3, H, W], crop_means [n]) on the host."""
    oh, ow = out
    prm = torch.from_numpy(np.ascontiguousarray(recs)).cuda()
    n = prm.shape[0]
    dst = torch.empty(n, 3, oh, ow, dtype=dtype, device="cuda")
    means = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    before = _lib.launches
    _lib.check(_lib.load().moco_augment_crops(pix.data_ptr(), pix.numel(), prm.data_ptr(), n, oh, ow, _norm(),
                                              dst.data_ptr(), _lib.dtype_code(dst), means.data_ptr(),
                                              _lib.cur_stream()), "moco_augment_crops")
    torch.cuda.synchronize()
    assert _lib.launches - before == 2
    return dst.cpu(), means.cpu().numpy()


def _resize(pix, recs, out, dtype=torch.float32):
    oh, ow = out
    prm = torch.from_numpy(np.ascontiguousarray(recs)).cuda()
    n = prm.shape[0]
    dst = torch.empty(n, 3, oh, ow, dtype=dtype, device="cuda")
    torch.cuda.synchronize()
    before = _lib.launches
    _lib.check(_lib.load().moco_resize_center_crops(pix.data_ptr(), pix.numel(), prm.data_ptr(), n, oh, ow, _norm(),
                                                    dst.data_ptr(), _lib.dtype_code(dst), _lib.cur_stream()),
               "moco_resize_center_crops")
    torch.cuda.synchronize()
    assert _lib.launches - before == 1
    return dst.cpu()


def _assert_exact(name, got, want):
    got = got.numpy()
    if not np.array_equal(got, want):
        bad = np.argwhere(got != want)
        i = tuple(bad[0])
        raise AssertionError(f"{name}: {len(bad)} of {got.size} values differ, first at {i}: kernel {got[i]!r} "
                             f"oracle {want[i]!r}")


def _check_means(name, recs, got, want):
    jit = (recs[:, MA.FLAGS] & AC.JITTER) != 0
    assert np.array_equal(got[jit], want[jit].astype(np.float32)), (name, got[jit], want[jit])
    assert (got[~jit] == 0).all(), (name, got[~jit])


def _check_augment(name, pix, recs, out, want, want_means):
    got, means = _augment(pix, recs, out)
    _assert_exact(name, got, want)
    _check_means(name, recs, means, want_means)
    bf, _ = _augment(pix, recs, out, torch.bfloat16)
    assert torch.equal(bf, got.to(torch.bfloat16)), name


@pytest.fixture(scope="module", autouse=True)
def _report():
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    print(f"\ntest_gpu_augment_exact: {time.time() - t0:.1f} s, peak device memory "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    torch.cuda.empty_cache()


AUG = {c.name: c for c in AC.aug_cases()}
RESIZE = {c.name: c for c in AC.resize_cases()}


@pytest.mark.parametrize("name", list(AUG))
def test_augment_case(name):
    case = AUG[name]
    img = case.image()
    pix, (off,) = _pack([img])
    want, want_means = AC.oracle_aug(case, img)
    _check_augment(name, pix, AC.records(case, off), case.out, want, want_means)


@pytest.mark.parametrize("name", list(RESIZE))
def test_resize_case(name):
    case = RESIZE[name]
    img = case.image()
    pix, (off,) = _pack([img])
    want = AC.oracle_resize(case, img)
    got = _resize(pix, AC.window_record(case, off), case.out)
    _assert_exact(name, got, want)
    assert torch.equal(_resize(pix, AC.window_record(case, off), case.out, torch.bfloat16), got.to(torch.bfloat16))


def test_65535_crops():
    """The grid limit: 65535 crops of 2 x 3 over 4 images, 8 boxes and the 5 flag variants, with factors drawn per
    crop; the oracle runs once per (image, box, variant) group."""
    n, out = 65535, (2, 3)
    images = [AC.image(40, 50, seed=500 + k) for k in range(4)]
    boxes = [(0, 0, 40, 50), (39, 49, 1, 1), (0, 49, 40, 1), (20, 25, 20, 25), (3, 5, 7, 11), (0, 0, 2, 3),
             (10, 0, 30, 50), (0, 10, 40, 40)]
    rng = np.random.default_rng(0)
    factors = np.concatenate([rng.uniform(0.6, 1.4, (n, 3)), rng.uniform(-0.5, 0.5, (n, 1))], 1).astype(np.float32)
    perms = list(itertools.permutations(range(4)))
    pix, offs = _pack(images)
    i = np.arange(n)
    img_of, box_of, var_of = i % 4, (i // 4) % 8, (i // 32) % len(AC.VARIANTS)
    recs = np.zeros((n, MA.WORDS), np.int32)
    for k in range(n):
        top, left, ch, cw = boxes[box_of[k]]
        flags = AC.VARIANTS[var_of[k]][0]
        recs[k, :MA.BRIGHTNESS] = [offs[img_of[k]], 0, 40, 50, top, left, ch, cw, flags,
                                   AC.order_word(perms[var_of[k] * 5 % 24])]
    recs[:, MA.BRIGHTNESS:] = factors.view(np.int32)
    want = np.zeros((n, 3) + out, np.float32)
    want_means = np.zeros(n, np.float32)
    for a, b, v in itertools.product(range(4), range(8), range(len(AC.VARIANTS))):
        sel = np.flatnonzero((img_of == a) & (box_of == b) & (var_of == v))
        top, left, ch, cw = boxes[b]
        box = np.broadcast_to(images[a][top:top + ch, left:left + cw], (len(sel), ch, cw, 3))
        o, m = O.augment(box, *out, AC.VARIANTS[v][0], int(recs[sel[0], MA.ORDER]), factors[sel], AC.NORM)
        want[sel], want_means[sel] = o, m
    _check_augment("65535 crops", pix, recs, out, want, want_means)


def test_sampler_batch():
    """512 crops of 256 images drawn by sample_crop_params as the loader draws them."""
    torch.manual_seed(11)
    images, recs = [], []
    for k in range(256):
        h, w = (375, 500) if k % 3 else (500, 375)
        images.append(AC.image(h, w, seed=1000 + k))
        recs.append(np.stack([MA.sample_crop_params(h, w, aug="CJ").numpy() for _ in range(2)]))
    pix, offs = _pack(images)
    recs = np.concatenate(recs)
    recs[:, MA.OFF_LO] = np.repeat(offs, 2)
    want = np.zeros((512, 3, 224, 224), np.float32)
    want_means = np.zeros(512, np.float32)
    for k in range(512):
        top, left, ch, cw, flags, order = (int(recs[k, j]) for j in (MA.TOP, MA.LEFT, MA.HEIGHT, MA.WIDTH,
                                                                          MA.FLAGS, MA.ORDER))
        box = images[k // 2][top:top + ch, left:left + cw][None]
        f = recs[k:k + 1, MA.BRIGHTNESS:].copy().view(np.float32)
        o, m = O.augment(box, 224, 224, flags, order, f, AC.NORM)
        want[k], want_means[k] = o[0], m[0]
    _check_augment("sampler batch", pix, recs, (224, 224), want, want_means)


def test_image_past_byte_2_to_the_32():
    """A 375 x 500 image at byte 2^32 + 3, ending at pixels_bytes: the crops of 224/whole,edges,1px on it."""
    case = AUG["224/whole,edges,1px"]
    img = case.image()
    need = BIG_OFFSET + img.nbytes + 2 * len(case.crops) * 3 * 224 * 224 * 4
    assert need < MAX_DEVICE_BYTES
    pix = torch.empty(BIG_OFFSET + img.nbytes, dtype=torch.uint8, device="cuda")
    pix[BIG_OFFSET:] = torch.from_numpy(img.reshape(-1)).cuda()
    want, want_means = AC.oracle_aug(case, img)
    _check_augment("past 2^32", pix, AC.records(case, BIG_OFFSET), case.out, want, want_means)
    del pix
    torch.cuda.empty_cache()
