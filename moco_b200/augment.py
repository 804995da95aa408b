"""The reference's data pipeline (train.py:92-125 with moco/dataset.py:7-35) with the augmentation on the GPU.

Workers only decode (``torchvision.io.decode_image``) and draw each crop's random parameters with torchvision's own
code, in the order the reference's ``Compose`` draws them; ``augment_two_crop`` sends the uint8 source pixels to the
device and one C call (``moco_augment_crops``, csrc/augment.cu) produces the [N, 6, H, W] batch ``MoCoStep`` takes.

The linear evaluation's loaders (eval.py:88-142) follow the same pattern: ``ImageFolderEval`` items carry one
decoded image and one record, ``augment_crops`` evaluates the train transform (a single crop per record) and
``resize_center_crops`` the validation transform, Resize -> CenterCrop -> Normalize, by one C call
(``moco_resize_center_crops``) that resamples only the centred window of the resized image.

Semantics: each crop equals torchvision's TENSOR implementation of the reference's transform applied to
``decoded_uint8 / 255`` in fp32 (``reference_crop`` / ``reference_resize_center_crop`` below), to fp32 rounding.  The
reference itself runs PIL on uint8, which rounds after the resize and after every jitter op, uses its own grayscale
weights and rounds the contrast mean to an integer; on the same draws the two differ by about one uint8 level on
average.

MoCo v2's augmentation (``aug="V2"``: RandomResizedCrop -> RandomApply(ColorJitter(0.4, 0.4, 0.4, 0.1), 0.8) ->
RandomGrayscale(0.2) -> RandomApply(GaussianBlur, 0.5) -> RandomHorizontalFlip -> Normalize) runs through
``moco_augment_crops_blur`` on 32-word records.  Its blur is torchvision's tensor ``GaussianBlur(23, (0.1, 2.0))``:
reflect padding and a fixed 23-tap kernel whose weights the workers compute with torchvision's own arithmetic
(``gaussian_half_kernel``), with sigma drawn by ``GaussianBlur.get_params`` on the torch RNG.  MoCo v2's own code
blurs with PIL's ``ImageFilter.GaussianBlur``, an approximation with no fixed kernel size, and draws sigma with
Python's ``random``; drawing on the torch RNG keeps ``seed_epoch``'s exact resume.  ``reference_crop`` rebuilds the
blur's kernel from the record's weights (the record holds no sigma), which are torchvision's bits.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch
import torchvision
from torchvision import transforms as T
from torchvision.transforms import functional as TF

from . import _lib

MEAN = (0.485, 0.456, 0.406)           # train.py:100
STD = (0.229, 0.224, 0.225)
RATIO = (3.0 / 4.0, 4.0 / 3.0)         # RandomResizedCrop's default aspect-ratio range
MAX_DOWNSCALE = 1000                   # a crop at most this many times wider than the output (include/moco_b200.h)

# one moco_aug_crop record (include/moco_b200.h) as 14 int32 words; the factors are stored by bit pattern
OFF_LO, OFF_HI, SRC_H, SRC_W, TOP, LEFT, HEIGHT, WIDTH, FLAGS, ORDER, BRIGHTNESS, CONTRAST, SATURATION, HUE = range(14)
WORDS = 14

# one moco_resize_window record (include/moco_b200.h) as 8 int32 words; words 0-3 are those of moco_aug_crop
RESIZED_H, RESIZED_W, WIN_TOP, WIN_LEFT = range(4, 8)
WIN_WORDS = 8

# one moco_aug_crop_blur record (MoCo v2) as 32 int32 words: the 14 above, the two switches and the half kernel
GRAY_LATE, BLUR, WEIGHTS = 14, 15, 16
V2_WORDS = 32
BLUR_KSIZE = 23                        # MoCo v2's blur as torchvision's tensor GaussianBlur(23, (0.1, 2.0))
BLUR_SIGMA = (0.1, 2.0)
AUGS = ("NULL", "CJ", "V2")

_JITTER = T.ColorJitter(0.4, 0.4, 0.4, 0.4)     # train.py:110; its ranges as torchvision stores them
_JITTER_V2 = T.ColorJitter(0.4, 0.4, 0.4, 0.1)  # MoCo v2's aug-plus


def _float_bits(values) -> list[int]:
    return torch.tensor(values, dtype=torch.float32).view(torch.int32).tolist()


def gaussian_half_kernel(ksize: int, sigma: float) -> list[float]:
    """kernel1d[ksize // 2:] of torchvision's _get_gaussian_kernel1d(ksize, sigma, float32, cpu), by the same torch
    ops, padded with zeros to 16 values: the weights of a moco_aug_crop_blur record."""
    half = (ksize - 1) * 0.5
    x = torch.linspace(-half, half, steps=ksize, dtype=torch.float32)
    pdf = torch.exp(-0.5 * (x / sigma).pow(2))
    k = pdf / pdf.sum()
    return k[ksize // 2:].tolist() + [0.0] * (16 - (ksize + 1) // 2)


def sample_crop_params(h: int, w: int, scale=(0.08, 1.0), aug: str = "CJ") -> torch.Tensor:
    """The random draws of one crop of an h x w image, made by torchvision's code on the global (or worker) RNG in
    the order the reference's Compose makes them (train.py:98-114): RandomResizedCrop.get_params, then for
    ``aug="CJ"`` the grayscale draw and ColorJitter.get_params, then the flip draw.  Returns the int32 [14] record
    with src_offset 0.  ``aug="V2"`` draws MoCo v2's Compose: RandomResizedCrop.get_params, RandomApply's draw and
    ColorJitter.get_params only if it applies, the grayscale draw, RandomApply's draw and GaussianBlur.get_params
    only if it applies, the flip draw; it returns the int32 [32] moco_aug_crop_blur record."""
    if aug not in AUGS:
        raise NotImplementedError(f"augmentation not supported: {aug}")
    top, left, ch, cw = T.RandomResizedCrop.get_params(torch.empty(1, 1, 1).expand(3, h, w), scale, RATIO)
    flags, order, factors = 0, 0, [1.0, 1.0, 1.0, 0.0]
    if aug == "V2":
        if not 0.8 < torch.rand(1):                                                  # RandomApply(p=0.8)
            fn_idx, b, c, s, hue = T.ColorJitter.get_params(_JITTER_V2.brightness, _JITTER_V2.contrast,
                                                            _JITTER_V2.saturation, _JITTER_V2.hue)
            flags |= _lib.AUG_JITTER
            order = sum(int(op) << (2 * k) for k, op in enumerate(fn_idx.tolist()))
            factors = [b, c, s, hue]
        if torch.rand(1) < 0.2:                                                      # RandomGrayscale(p=0.2)
            flags |= _lib.AUG_GRAY
        blur, weights = 0, [0.0] * 16
        if not 0.5 < torch.rand(1):                                                  # RandomApply(p=0.5)
            blur, weights = 1, gaussian_half_kernel(BLUR_KSIZE, T.GaussianBlur.get_params(*BLUR_SIGMA))
        if torch.rand(1) < 0.5:                                                      # RandomHorizontalFlip()
            flags |= _lib.AUG_FLIP
        return torch.tensor([0, 0, h, w, top, left, ch, cw, flags, order] + _float_bits(factors) + [1, blur] +
                            _float_bits(weights), dtype=torch.int32)
    if aug == "CJ":
        if torch.rand(1) < 0.2:                                                      # RandomGrayscale(p=0.2)
            flags |= _lib.AUG_GRAY
        fn_idx, b, c, s, hue = T.ColorJitter.get_params(_JITTER.brightness, _JITTER.contrast, _JITTER.saturation,
                                                        _JITTER.hue)
        flags |= _lib.AUG_JITTER
        order = sum(int(op) << (2 * k) for k, op in enumerate(fn_idx.tolist()))
        factors = [b, c, s, hue]
    if torch.rand(1) < 0.5:                                                          # RandomHorizontalFlip()
        flags |= _lib.AUG_FLIP
    return torch.tensor([0, 0, h, w, top, left, ch, cw, flags, order] + _float_bits(factors), dtype=torch.int32)


def validate_params(params: torch.Tensor, pixels_bytes: int, out_w: int | None = None) -> None:
    """Raise ValueError unless every record of the int32 [n, 14] ``params`` describes a crop inside its image, inside
    a buffer of ``pixels_bytes`` bytes, with a permutation as jitter order and factors in ColorJitter's domain."""
    p = np.asarray(params.detach().cpu(), dtype=np.int32)
    if p.ndim != 2 or p.shape[1] != WORDS:
        raise ValueError(f"crop parameters must be int32 [n, {WORDS}], got {tuple(p.shape)}")
    q = p.astype(np.int64)
    off = (q[:, OFF_LO] & 0xFFFFFFFF) | (q[:, OFF_HI] << 32)
    h, w, top, left, ch, cw = (q[:, k] for k in (SRC_H, SRC_W, TOP, LEFT, HEIGHT, WIDTH))
    f = p[:, BRIGHTNESS:].copy().view(np.float32)

    def bad(mask, what):
        if mask.any():
            raise ValueError(f"crop parameters: {what} (record {int(np.flatnonzero(mask)[0])})")

    bad((h < 1) | (w < 1), "image size below 1")
    bad((off < 0) | (off + h * w * 3 > pixels_bytes), "image outside the pixel buffer")
    bad((ch < 1) | (cw < 1), "crop size below 1")
    bad((top < 0) | (left < 0) | (top + ch > h) | (left + cw > w), "crop box outside its image")
    if out_w is not None:
        bad(cw > MAX_DOWNSCALE * out_w, f"crop more than {MAX_DOWNSCALE} times wider than the output")
    flags, order = q[:, FLAGS], q[:, ORDER]
    bad((flags & ~(_lib.AUG_GRAY | _lib.AUG_FLIP | _lib.AUG_JITTER)) != 0, "unknown flag bits")
    jit = (flags & _lib.AUG_JITTER) != 0
    ops = np.stack([(order >> (2 * k)) & 3 for k in range(4)], axis=1)
    perm = (order >= 0) & (order < 256) & (np.sort(ops, axis=1) == np.arange(4)).all(axis=1)
    bad(jit & ~perm, "jitter order is not a permutation of the four ops")
    bad(~np.isfinite(f).all(axis=1), "non-finite factor")
    bad(jit & ((f[:, :3] < 0).any(axis=1) | (np.abs(f[:, 3]) > 0.5)), "factor out of range")


def validate_params_v2(params: torch.Tensor, pixels_bytes: int, out_w: int | None = None,
                       ksize: int = BLUR_KSIZE) -> None:
    """Raise ValueError unless every record of the int32 [n, 32] ``params`` passes ``validate_params`` on its first
    14 words, has 0 or 1 as its two switches, and weights that are finite, in [0, 1] and zero past ksize // 2."""
    p = np.asarray(params.detach().cpu(), dtype=np.int32)
    if p.ndim != 2 or p.shape[1] != V2_WORDS:
        raise ValueError(f"crop parameters must be int32 [n, {V2_WORDS}], got {tuple(p.shape)}")
    if not (3 <= ksize <= 31 and ksize % 2):
        raise ValueError(f"crop parameters: the blur's ksize must be odd and in [3, 31], got {ksize}")
    validate_params(torch.from_numpy(np.ascontiguousarray(p[:, :WORDS])), pixels_bytes, out_w)
    wts = p[:, WEIGHTS:].copy().view(np.float32)

    def bad(mask, what):
        if mask.any():
            raise ValueError(f"crop parameters: {what} (record {int(np.flatnonzero(mask)[0])})")

    bad((p[:, GRAY_LATE] != 0) & (p[:, GRAY_LATE] != 1), "gray_after_jitter is not 0 or 1")
    bad((p[:, BLUR] != 0) & (p[:, BLUR] != 1), "blur is not 0 or 1")
    bad(~np.isfinite(wts).all(axis=1), "non-finite blur weight")
    bad(((wts < 0) | (wts > 1)).any(axis=1), "blur weight outside [0, 1]")
    bad((wts[:, ksize // 2 + 1:] != 0).any(axis=1), f"blur weight past ksize // 2 = {ksize // 2}")


def _validate_records(params, pixels_bytes, out_w=None):
    """validate_params or validate_params_v2, by the records' width."""
    if params.dim() == 2 and params.shape[1] == V2_WORDS:
        validate_params_v2(params, pixels_bytes, out_w)
    else:
        validate_params(params, pixels_bytes, out_w)


def resize_window_params(h: int, w: int, resize: int = 256, out: int = 224) -> torch.Tensor:
    """The int32 [8] moco_resize_window record (src_offset 0) of Resize(resize) -> CenterCrop(out) on an h x w image,
    with torchvision's arithmetic: the short side becomes ``resize`` and the long side int(resize * long / short)
    (transforms.functional._compute_resized_output_size); the window starts at int(round((resized - out) / 2.0)),
    Python's round half to even (center_crop).  Raises ValueError when the window does not fit inside the resized
    image: center_crop would zero-pad there, which the kernel does not do (it never happens at 256 / 224)."""
    if min(h, w, resize, out) < 1:
        raise ValueError(f"resize_window_params: sizes must be >= 1 (h={h} w={w} resize={resize} out={out})")
    short, long = (w, h) if w <= h else (h, w)
    new_long = int(resize * long / short)
    rh, rw = (new_long, resize) if w <= h else (resize, new_long)
    if rh < out or rw < out:
        raise ValueError(f"resize_window_params: a {out} x {out} window does not fit in the {rh} x {rw} resized image")
    top, left = int(round((rh - out) / 2.0)), int(round((rw - out) / 2.0))
    return torch.tensor([0, 0, h, w, rh, rw, top, left], dtype=torch.int32)


def validate_windows(params: torch.Tensor, pixels_bytes: int, out_h: int, out_w: int, resize: int | None = None) -> None:
    """Raise ValueError unless every record of the int32 [n, 8] ``params`` describes an image inside a buffer of
    ``pixels_bytes`` bytes and an out_h x out_w window inside its resized image, within the kernel's downscale limit
    (and, given ``resize``, a resized short side of ``resize``)."""
    p = np.asarray(params.detach().cpu(), dtype=np.int32)
    if p.ndim != 2 or p.shape[1] != WIN_WORDS:
        raise ValueError(f"resize windows must be int32 [n, {WIN_WORDS}], got {tuple(p.shape)}")
    q = p.astype(np.int64)
    off = (q[:, OFF_LO] & 0xFFFFFFFF) | (q[:, OFF_HI] << 32)
    h, w, rh, rw, top, left = (q[:, k] for k in (SRC_H, SRC_W, RESIZED_H, RESIZED_W, WIN_TOP, WIN_LEFT))

    def bad(mask, what):
        if mask.any():
            raise ValueError(f"resize windows: {what} (record {int(np.flatnonzero(mask)[0])})")

    bad((h < 1) | (w < 1), "image size below 1")
    bad((off < 0) | (off + h * w * 3 > pixels_bytes), "image outside the pixel buffer")
    bad((rh < 1) | (rw < 1), "resized size below 1")
    bad((top < 0) | (left < 0) | (top + out_h > rh) | (left + out_w > rw), "window outside the resized image")
    bad(w > MAX_DOWNSCALE * rw, f"image more than {MAX_DOWNSCALE} times wider than its resized width")
    if resize is not None:
        bad(np.minimum(rh, rw) != resize, f"resized short side is not {resize}")


def pack_images(images, records) -> tuple[torch.Tensor, torch.Tensor]:
    """[uint8 HWC image], [int32 [k, words] records of that image] -> (uint8 [sum of h*w*3] packed pixels, int32
    [sum of k, words] records with each image's byte offset filled in)."""
    sizes = [img.numel() for img in images]
    offsets = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    pixels = torch.cat([img.reshape(-1) for img in images])
    params = torch.cat(list(records)).clone()
    off = np.repeat(offsets, [r.shape[0] for r in records])
    params[:, OFF_LO] = torch.from_numpy((off & 0xFFFFFFFF).astype(np.uint32).view(np.int32))
    params[:, OFF_HI] = torch.from_numpy((off >> 32).astype(np.int32))
    return pixels, params


class ImageFolderTwoCrop(torchvision.datasets.ImageFolder):
    """moco/dataset.py's ImageFolderInstance(two_crop=True) with train.py's transform, minus the pixel work: an item
    is (decoded uint8 HWC image, int32 [2, 14] parameters of its two crops, target), [2, 32] for ``aug="V2"``.  Use
    ``collate_fn`` as the DataLoader's collate_fn and ``augment_two_crop`` on what it yields."""

    def __init__(self, root, scale=(0.08, 1.0), aug: str = "CJ"):
        if aug not in AUGS:
            raise NotImplementedError(f"augmentation not supported: {aug}")
        super().__init__(root)
        self.scale = tuple(scale)
        self.aug = aug

    def __getitem__(self, index):
        path, target = self.samples[index]
        img = torchvision.io.decode_image(path, mode=torchvision.io.ImageReadMode.RGB)
        hwc = img.permute(1, 2, 0).contiguous()
        h, w = hwc.shape[0], hwc.shape[1]
        params = torch.stack([sample_crop_params(h, w, self.scale, self.aug) for _ in range(2)])   # crop 1, then 2
        return hwc, params, target

    @staticmethod
    def collate_fn(items):
        """[(hwc, params, target)] -> (uint8 [sum of h*w*3] packed pixels, int32 [2N, 14] params with each image's
        byte offset filled in, int64 [N] targets).  DataLoader(pin_memory=True) pins all three."""
        pixels, params = pack_images([it[0] for it in items], [it[1] for it in items])
        _validate_records(params, pixels.numel())
        return pixels, params, torch.tensor([it[2] for it in items], dtype=torch.int64)


class ImageFolderEval(torchvision.datasets.ImageFolder):
    """One split of eval.py's loaders (eval.py:88-142) minus the pixel work: an item is (decoded uint8 HWC image,
    int32 [1, words] record, target, dataset index).  ``train=True`` items carry one ``sample_crop_params`` record,
    drawn in the order of eval.py's train Compose (RandomResizedCrop(224, scale) [-> RandomGrayscale -> ColorJitter
    for ``aug="CJ"``] -> RandomHorizontalFlip), ``aug="NULL"`` by default as in eval.py; use ``augment_crops`` on the
    collated batch.  ``train=False`` items carry one ``resize_window_params`` record (Resize(resize) ->
    CenterCrop(out)); use ``resize_center_crops``.  Pass ``ds.collate_fn`` as the DataLoader's collate_fn."""

    def __init__(self, root, train: bool, scale=(0.08, 1.0), aug: str = "NULL", resize: int = 256, out: int = 224):
        if aug not in ("CJ", "NULL"):
            raise NotImplementedError(f"augmentation not supported: {aug}")
        super().__init__(root)
        self.train = bool(train)
        self.scale = tuple(scale)
        self.aug = aug
        self.resize = int(resize)
        self.out = int(out)

    def __getitem__(self, index):
        path, target = self.samples[index]
        img = torchvision.io.decode_image(path, mode=torchvision.io.ImageReadMode.RGB)
        hwc = img.permute(1, 2, 0).contiguous()
        h, w = hwc.shape[0], hwc.shape[1]
        if self.train:
            rec = sample_crop_params(h, w, self.scale, self.aug)
        else:
            rec = resize_window_params(h, w, self.resize, self.out)
        return hwc, rec.unsqueeze(0), target, index

    def collate_fn(self, items):
        """[(hwc, record, target, index)] -> (uint8 packed pixels, int32 [N, words] records with byte offsets filled
        in and validated, int64 [N] targets, int64 [N] dataset indices).  DataLoader(pin_memory=True) pins them."""
        pixels, params = pack_images([it[0] for it in items], [it[1] for it in items])
        if self.train:
            validate_params(params, pixels.numel(), self.out)
        else:
            validate_windows(params, pixels.numel(), self.out, self.out, self.resize)
        return (pixels, params, torch.tensor([it[2] for it in items], dtype=torch.int64),
                torch.tensor([it[3] for it in items], dtype=torch.int64))


def _device(device, what):
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if dev.type != "cuda":
        raise RuntimeError(f"moco_b200: {what} runs on CUDA only; there is no CPU fallback")
    return dev


def augment_crops(batch, out_size=224, mean=MEAN, std=STD, dtype=torch.bfloat16, device=None) -> torch.Tensor:
    """(pixels, params, ...) with int32 [n, 14] crop records -> [n, 3, H, W], one crop per record, computed on
    ``device`` (default: the current CUDA device) by one C call (moco_augment_crops).  The pixels and records are
    copied with non_blocking=True (asynchronous from pinned memory).  int32 [n, 32] records (``aug="V2"``) go to
    moco_augment_crops_blur with the blur's kernel size BLUR_KSIZE."""
    pixels, params = batch[0], batch[1]
    out_h, out_w = (out_size, out_size) if isinstance(out_size, int) else tuple(out_size)
    _validate_records(params, pixels.numel(), out_w)
    dev = _device(device, "augment_crops")
    if pixels.dtype != torch.uint8:
        raise TypeError("augment_crops: pixels must be uint8")
    pix = pixels.reshape(-1).to(dev, non_blocking=True)
    prm = params.to(torch.int32).contiguous().to(dev, non_blocking=True)
    n = prm.shape[0]
    out = torch.empty(n, 3, out_h, out_w, dtype=dtype, device=dev)
    means = torch.empty(max(n, 1), dtype=torch.float32, device=dev)
    norm = (ctypes.c_float * 6)(*mean, *std)
    with torch.cuda.device(dev):
        lib = _lib.load()
        if prm.shape[1] == V2_WORDS:
            _lib.check(lib.moco_augment_crops_blur(pix.data_ptr(), pix.numel(), prm.data_ptr(), n, out_h, out_w,
                                                   BLUR_KSIZE, norm, out.data_ptr(), _lib.dtype_code(out),
                                                   means.data_ptr(), _lib.cur_stream()), "moco_augment_crops_blur")
        else:
            _lib.check(lib.moco_augment_crops(pix.data_ptr(), pix.numel(), prm.data_ptr(), n, out_h, out_w, norm,
                                              out.data_ptr(), _lib.dtype_code(out), means.data_ptr(),
                                              _lib.cur_stream()), "moco_augment_crops")
    return out


def augment_two_crop(batch, out_size=224, mean=MEAN, std=STD, dtype=torch.bfloat16, device=None) -> torch.Tensor:
    """(pixels, params[, targets]) from ImageFolderTwoCrop.collate_fn -> the [N, 6, H, W] batch of the reference's
    loader (dataset.py:31-33), computed on ``device`` (default: the current CUDA device) by one C call: the
    ``augment_crops`` batch of the 2N crops, viewed as N pairs."""
    params = batch[1]
    if params.shape[0] % 2:
        raise ValueError("augment_two_crop: an odd number of crop records")
    out = augment_crops(batch, out_size, mean, std, dtype, device)
    n, _, out_h, out_w = out.shape
    return out.view(n // 2, 6, out_h, out_w)


def seed_epoch(loader, rng_seed: int, epoch: int, rank: int) -> None:
    """Make epoch ``epoch``'s crop draws a function of (rng_seed, epoch, rank) alone: set the sampler's epoch and
    seed the generator the next iterator draws its workers' seeds from -- or, without workers, the main process's
    CPU generator, on which the dataset then draws.  ``loader`` needs its own ``generator`` and a sampler with
    ``set_epoch``; workers must not be persistent, so that every epoch starts them afresh from that generator."""
    loader.sampler.set_epoch(epoch)                                                      # train.py:213, eval.py:235
    seed = int(np.random.SeedSequence([rng_seed % 2 ** 64, epoch, rank]).generate_state(1, np.uint64)[0] >> 1)
    loader.generator.manual_seed(seed)
    if loader.num_workers == 0:
        torch.default_generator.manual_seed(seed)


def prefetch_pixels(batches, device=None):
    """Yield each (pixels, params, ...) batch of ``batches`` with its pixels copied to ``device`` (default: the
    current CUDA device) on a dedicated copy stream, so that the copy of batch i + 1 -- issued when the caller asks
    for it, after queueing its work on batch i -- runs while that work does, instead of waiting for it on the
    compute stream.  The current stream waits for the copy before anything it queues after the yield, and the
    caching allocator keeps the device pixels until that stream is done with them.  The records stay on the host;
    ``augment_crops`` / ``augment_two_crop`` take the batch as it is."""
    dev = _device(device, "prefetch_pixels")
    copy = torch.cuda.Stream(dev)
    for batch in batches:
        main = torch.cuda.current_stream(dev)
        with torch.cuda.stream(copy):
            pixels = batch[0].to(dev, non_blocking=True)
        main.wait_stream(copy)
        pixels.record_stream(main)
        yield (pixels,) + tuple(batch[1:])


def resize_center_crops(batch, resize=256, out=224, mean=MEAN, std=STD, dtype=torch.bfloat16,
                        device=None) -> torch.Tensor:
    """(pixels, windows, ...) from ``ImageFolderEval(train=False).collate_fn`` -> the [n, 3, out, out] batch of
    eval.py's validation transform (Resize(resize) -> CenterCrop(out) -> ToTensor -> Normalize), computed on
    ``device`` (default: the current CUDA device) by one C call (moco_resize_center_crops, one launch).  The pixels
    and records are copied with non_blocking=True."""
    pixels, params = batch[0], batch[1]
    validate_windows(params, pixels.numel(), out, out, resize)
    dev = _device(device, "resize_center_crops")
    if pixels.dtype != torch.uint8:
        raise TypeError("resize_center_crops: pixels must be uint8")
    pix = pixels.reshape(-1).to(dev, non_blocking=True)
    prm = params.to(torch.int32).contiguous().to(dev, non_blocking=True)
    n = prm.shape[0]
    dst = torch.empty(n, 3, out, out, dtype=dtype, device=dev)
    norm = (ctypes.c_float * 6)(*mean, *std)
    with torch.cuda.device(dev):
        lib = _lib.load()
        _lib.check(lib.moco_resize_center_crops(pix.data_ptr(), pix.numel(), prm.data_ptr(), n, out, out, norm,
                                                dst.data_ptr(), _lib.dtype_code(dst), _lib.cur_stream()),
                   "moco_resize_center_crops")
    return dst


def reference_crop(hwc_uint8: torch.Tensor, record, out_size=224, mean=MEAN, std=STD,
                   ksize: int = BLUR_KSIZE) -> torch.Tensor:
    """What the kernel computes for one crop, with torchvision's functional tensor ops on the CPU:
    [3, H, W] fp32 from a uint8 HWC image and one int32 [14] record (train.py:106-114 with the record's draws).
    A 32-word record is MoCo v2's: the grayscale after the jitter when gray_after_jitter is set, and with blur set
    torchvision's tensor gaussian_blur of size ``ksize`` with the kernel rebuilt from the record's weights."""
    r = [int(v) for v in record]
    f = torch.tensor(r[BRIGHTNESS:WORDS], dtype=torch.int32).view(torch.float32).tolist()
    v2 = len(r) == V2_WORDS
    gray_late = v2 and r[GRAY_LATE] != 0
    out_hw = [out_size, out_size] if isinstance(out_size, int) else list(out_size)
    x = hwc_uint8.permute(2, 0, 1).float() / 255
    x = TF.resized_crop(x, r[TOP], r[LEFT], r[HEIGHT], r[WIDTH], out_hw, antialias=True)
    if r[FLAGS] & _lib.AUG_GRAY and not gray_late:
        x = TF.rgb_to_grayscale(x, 3)
    if r[FLAGS] & _lib.AUG_JITTER:
        ops = (TF.adjust_brightness, TF.adjust_contrast, TF.adjust_saturation, TF.adjust_hue)
        for k in range(4):
            op = (r[ORDER] >> (2 * k)) & 3
            x = ops[op](x, f[op])
    if r[FLAGS] & _lib.AUG_GRAY and gray_late:
        x = TF.rgb_to_grayscale(x, 3)
    if v2 and r[BLUR]:
        half = torch.tensor(r[WEIGHTS:], dtype=torch.int32).view(torch.float32)[:ksize // 2 + 1]
        k1d = torch.cat([half.flip(0)[:-1], half])
        k2d = torch.mm(k1d[:, None], k1d[None, :]).expand(3, 1, ksize, ksize)
        x = torch.nn.functional.pad(x[None], [ksize // 2] * 4, mode="reflect")
        x = torch.nn.functional.conv2d(x, k2d, groups=3)[0]
    if r[FLAGS] & _lib.AUG_FLIP:
        x = TF.hflip(x)
    return TF.normalize(x, list(mean), list(std))


def reference_compose(aug: str = "CJ", scale=(0.08, 1.0), out_size=224):
    """train.py:98-114's transform as tensor ops on a float [3, h, w] image in [0, 1] (ToTensor already applied);
    ``aug="V2"`` MoCo v2's, with torchvision's tensor GaussianBlur(23, (0.1, 2.0))."""
    if aug == "V2":
        ts = [T.RandomResizedCrop(out_size, scale=scale), T.RandomApply([T.ColorJitter(0.4, 0.4, 0.4, 0.1)], p=0.8),
              T.RandomGrayscale(p=0.2), T.RandomApply([T.GaussianBlur(BLUR_KSIZE, BLUR_SIGMA)], p=0.5),
              T.RandomHorizontalFlip()]
    elif aug == "NULL":
        ts = [T.RandomResizedCrop(out_size, scale=scale), T.RandomHorizontalFlip()]
    else:
        ts = [T.RandomResizedCrop(out_size, scale=scale), T.RandomGrayscale(p=0.2), T.ColorJitter(0.4, 0.4, 0.4, 0.4),
              T.RandomHorizontalFlip()]
    return T.Compose(ts + [T.Normalize(mean=MEAN, std=STD)])


def reference_resize_center_crop(hwc_uint8: torch.Tensor, record, out=224, mean=MEAN, std=STD) -> torch.Tensor:
    """What moco_resize_center_crops computes for one image, with torchvision's functional tensor ops on the CPU in
    fp32: [3, out, out] from a uint8 HWC image and its int32 [8] record (eval.py:111-116 with the record's resized
    size)."""
    r = [int(v) for v in record]
    x = hwc_uint8.permute(2, 0, 1).float() / 255
    x = TF.resize(x, [r[RESIZED_H], r[RESIZED_W]], antialias=True)
    x = TF.center_crop(x, [out, out])
    return TF.normalize(x, list(mean), list(std))


def reference_val_compose(resize=256, out=224):
    """eval.py:111-116's validation transform as tensor ops on a float [3, h, w] image in [0, 1]."""
    return T.Compose([T.Resize(resize), T.CenterCrop(out), T.Normalize(mean=MEAN, std=STD)])
