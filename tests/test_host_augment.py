"""Host side of the GPU augmentation (moco_b200/augment.py), no GPU needed: the parameter sampler plus torchvision's
functional ops reproduce the reference's Compose bit for bit, ImageFolderTwoCrop packs what decode_image returns with
consistent offsets and records, malformed records raise ValueError, and the example trainer's data flags parse."""
import importlib.util
import os

import numpy as np
import pytest
import torch
import torchvision

from moco_b200 import _lib
from moco_b200 import augment as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _image(h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8)


@pytest.mark.parametrize("aug", ["CJ", "NULL"])
@pytest.mark.parametrize("hw", [(375, 500), (30, 600), (600, 30)])
def test_sampler_and_functional_ops_equal_compose(aug, hw):
    """50 seeds: sample_crop_params drawn on the global RNG + reference_crop == train.py's Compose on the same RNG.
    30 x 600 and 600 x 30 force RandomResizedCrop.get_params' fallback center crop."""
    img = _image(*hw, seed=hw[0])
    x = img.permute(2, 0, 1).float() / 255
    comp = A.reference_compose(aug)
    for seed in range(50):
        torch.manual_seed(seed)
        ref = comp(x)
        torch.manual_seed(seed)
        rec = A.sample_crop_params(*hw, aug=aug)
        assert torch.equal(A.reference_crop(img, rec), ref), (aug, hw, seed)
        assert bool(rec[A.FLAGS] & _lib.AUG_JITTER) == (aug == "CJ")


def test_fallback_center_crop_is_drawn_for_extreme_aspect_ratios():
    torch.manual_seed(0)
    rec = A.sample_crop_params(30, 600, aug="NULL")
    assert (int(rec[A.HEIGHT]), int(rec[A.WIDTH]), int(rec[A.TOP])) == (30, 40, 0)
    assert int(rec[A.LEFT]) == (600 - 40) // 2


def _jpeg_folder(root, sizes, classes=2):
    for c in range(classes):
        os.makedirs(os.path.join(root, "train", f"class{c}"), exist_ok=True)
    for i, (h, w) in enumerate(sizes):
        img = _image(h, w, seed=100 + i).permute(2, 0, 1).contiguous()
        data = torchvision.io.encode_jpeg(img, quality=90)
        with open(os.path.join(root, "train", f"class{i % classes}", f"img{i:03d}.jpg"), "wb") as f:
            f.write(data.numpy().tobytes())
    return os.path.join(root, "train")


def test_image_folder_packs_decoded_pixels_and_consistent_records(tmp_path):
    sizes = [(64, 80), (97, 61), (120, 120), (33, 250)]
    root = _jpeg_folder(str(tmp_path), sizes)
    ds = A.ImageFolderTwoCrop(root, scale=(0.2, 1.0), aug="CJ")
    torch.manual_seed(3)
    items = [ds[i] for i in range(len(ds))]
    pixels, params, targets = A.ImageFolderTwoCrop.collate_fn(items)
    assert pixels.dtype == torch.uint8 and params.dtype == torch.int32 and params.shape == (2 * len(ds), A.WORDS)
    assert targets.tolist() == [t for _, t in ds.samples]
    off = 0
    for n, (path, _) in enumerate(ds.samples):
        dec = torchvision.io.decode_image(path, mode=torchvision.io.ImageReadMode.RGB).permute(1, 2, 0)
        h, w = dec.shape[:2]
        assert torch.equal(pixels[off:off + h * w * 3].view(h, w, 3), dec)
        for c in range(2):
            r = params[2 * n + c].tolist()
            assert r[A.OFF_LO] == off and r[A.OFF_HI] == 0 and (r[A.SRC_H], r[A.SRC_W]) == (h, w)
            assert 0 <= r[A.TOP] and r[A.TOP] + r[A.HEIGHT] <= h and 0 <= r[A.LEFT] and r[A.LEFT] + r[A.WIDTH] <= w
            assert sorted((r[A.ORDER] >> (2 * k)) & 3 for k in range(4)) == [0, 1, 2, 3]
        off += h * w * 3
    assert off == pixels.numel()


def test_loader_yields_packed_batches_without_workers(tmp_path):
    root = _jpeg_folder(str(tmp_path), [(50 + 7 * i, 70 - 3 * i) for i in range(6)])
    ds = A.ImageFolderTwoCrop(root, aug="NULL")
    loader = torch.utils.data.DataLoader(ds, batch_size=4, num_workers=0, drop_last=True,
                                         collate_fn=A.ImageFolderTwoCrop.collate_fn)
    batches = list(loader)
    assert len(batches) == 1
    pixels, params, targets = batches[0]
    assert params.shape == (8, A.WORDS) and targets.shape == (4,)
    assert int(params[-1, A.OFF_LO]) + int(params[-1, A.SRC_H]) * int(params[-1, A.SRC_W]) * 3 == pixels.numel()
    A.validate_params(params, pixels.numel(), 224)


def _good():
    torch.manual_seed(0)
    return torch.stack([A.sample_crop_params(100, 120), A.sample_crop_params(100, 120)]), 100 * 120 * 3


def _f32(v):
    return int(torch.tensor([v], dtype=torch.float32).view(torch.int32))


@pytest.mark.parametrize("word,value,match", [
    (A.OFF_LO, 3, "outside the pixel buffer"),
    (A.OFF_HI, -1, "outside the pixel buffer"),
    (A.SRC_H, 0, "image size"),
    (A.SRC_W, 121, "outside the pixel buffer"),
    (A.HEIGHT, 0, "crop size"),
    (A.WIDTH, -4, "crop size"),
    (A.TOP, -1, "crop box"),
    (A.LEFT, 120, "crop box"),
    (A.FLAGS, 8, "flag bits"),
    (A.ORDER, 0b00011011 & ~0b11 | 0b01, "permutation"),
    (A.ORDER, 256 + 0b11100100, "permutation"),
    (A.CONTRAST, _f32(-0.1), "out of range"),
    (A.HUE, _f32(0.6), "out of range"),
    (A.SATURATION, _f32(float("nan")), "non-finite"),
])
def test_malformed_records_raise_value_error(word, value, match):
    params, nbytes = _good()
    A.validate_params(params, nbytes, 224)
    bad = params.clone()
    bad[1, word] = value
    if word == A.TOP:
        bad[1, A.HEIGHT] = 1
    if word == A.LEFT:
        bad[1, A.WIDTH] = 1
    with pytest.raises(ValueError, match=match):
        A.validate_params(bad, nbytes, 224)


def test_crop_far_wider_than_the_output_is_refused():
    params, _ = _good()
    params[0, A.SRC_W] = params[0, A.WIDTH] = 1001 * 4
    params[0, A.LEFT] = 0
    A.validate_params(params[:1], 10 ** 9)
    with pytest.raises(ValueError, match="wider"):
        A.validate_params(params[:1], 10 ** 9, 4)


def test_augment_two_crop_refuses_a_cpu_device():
    params, nbytes = _good()
    with pytest.raises(RuntimeError, match="CUDA only"):
        A.augment_two_crop((torch.zeros(nbytes, dtype=torch.uint8), params), device="cpu")


def test_augment_entry_validates_its_arguments_without_a_gpu():
    import ctypes
    lib = _lib.load()
    norm = (ctypes.c_float * 6)(*A.MEAN, *A.STD)
    addr = 0x7f0000001000
    args = [addr, 1000, addr + 0x1000, 2, 224, 224, norm, addr + 0x2000, _lib.MOCO_BF16, addr + 0x3000, None]
    for k, v in ((0, None), (1, 0), (2, addr + 4), (8, 7), (9, addr + 2), (4, 0), (5, 1025), (3, 70000)):
        a = list(args)
        a[k] = v
        assert lib.moco_augment_crops(*a) == -1, (k, v)
        assert b"moco_augment_crops" in lib.moco_last_error()
    zero_std = (ctypes.c_float * 6)(*A.MEAN, 0.2, 0.0, 0.2)
    a = list(args)
    a[6] = zero_std
    assert lib.moco_augment_crops(*a) == -1 and b"std" in lib.moco_last_error()
    a = list(args)
    a[3] = 0
    assert lib.moco_augment_crops(*a) == 0          # no crops: nothing is launched


def test_header_flag_constants_match():
    import re
    text = open(os.path.join(ROOT, "include", "moco_b200.h")).read()
    enum = {m.group(1): int(m.group(2)) for m in re.finditer(r"\b(MOCO_AUG_[A-Z]+)\s*=\s*(\d+)", text)}
    assert enum == {"MOCO_AUG_GRAY": _lib.AUG_GRAY, "MOCO_AUG_FLIP": _lib.AUG_FLIP, "MOCO_AUG_JITTER": _lib.AUG_JITTER}


def test_example_trainer_parses_the_data_flags():
    spec = importlib.util.spec_from_file_location("train_moco_example_aug", os.path.join(ROOT, "examples", "train_moco.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    a = mod.parse_args([])
    assert (a.data_dir, a.crop, a.aug, a.num_workers) == ("", 0.08, "CJ", 4)
    a = mod.parse_args(["--data-dir", "/d", "--crop", "0.2", "--aug", "NULL", "--num-workers", "8"])
    assert (a.data_dir, a.crop, a.aug, a.num_workers) == ("/d", 0.2, "NULL", 8)
    with pytest.raises(SystemExit):
        mod.parse_args(["--aug", "RA"])


def test_example_trainer_loader_uses_the_reference_sampling(tmp_path):
    spec = importlib.util.spec_from_file_location("train_moco_example_aug2", os.path.join(ROOT, "examples", "train_moco.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    _jpeg_folder(str(tmp_path), [(40, 40)] * 5)
    args = mod.parse_args(["--data-dir", str(tmp_path), "--batch-size", "2", "--num-workers", "0"])
    loader = mod.make_loader(args, world=1)
    assert loader.drop_last and len(loader) == 2
    pixels, params, _ = next(iter(loader))
    assert params.shape == (4, A.WORDS) and pixels.numel() == 2 * 40 * 40 * 3
    assert np.all(params[:, A.SRC_H].numpy() == 40)
