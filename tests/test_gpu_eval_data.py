"""The linear evaluation's data path on the GPU: moco_resize_center_crops (csrc/augment.cu) against torchvision's
tensor ops (moco_b200.augment.reference_resize_center_crop, fp32 on the CPU) for upsampled, identity-resized,
half-to-even-offset and column-chunked sources, two resize / crop pairs and a 256-image batch of mixed sizes; bf16 =
rounded fp32, run-to-run bit identity and one launch per call; augment_crops with one crop per record; and a JPEG
folder end to end through the loaders and examples/eval_linear.py."""
import gc
import importlib.util
import math
import os

import pytest
import torch
import torchvision

from moco_b200 import _lib
from moco_b200 import augment as A

pytestmark = pytest.mark.gpu
BOUND = 1e-4          # max |kernel - torchvision| in normalised units (as test_gpu_augment)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def _release_what_this_module_cached():
    """These tests crop sources up to 4000 x 3000 and run a ResNet-50 through pinned-memory DataLoaders.  Afterwards,
    hand the device memory and pinned host memory they left in torch's caches back to the driver, so that the tests
    after them in the same process run with the memory they would have had without them."""
    yield
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch._C._host_emptyCache()


def _image(h, w, seed):
    g = torch.Generator().manual_seed(seed)
    base = torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.int32)
    yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    smooth = torch.stack([(yy * 255) // max(h - 1, 1), (xx * 255) // max(w - 1, 1), ((yy + xx) * 7) % 256], -1)
    img = ((base + 3 * smooth) // 4).to(torch.uint8)
    img[-2:, -2:] = 255
    return img.contiguous()


def _windows(images, resize, out):
    recs = [A.resize_window_params(img.shape[0], img.shape[1], resize, out)[None] for img in images]
    return A.pack_images(images, recs)


def _check(images, resize=256, out=224):
    pixels, params = _windows(images, resize, out)
    got = A.resize_center_crops((pixels, params), resize, out, dtype=torch.float32).cpu()
    assert got.shape == (len(images), 3, out, out)
    worst = 0.0
    for i, img in enumerate(images):
        ref = A.reference_resize_center_crop(img, params[i], out)
        worst = max(worst, float((got[i] - ref).abs().max()))
    print(f"max |diff| = {worst:.3g}")
    assert worst <= BOUND, worst
    return worst


SIZES = [(100, 150), (150, 100), (255, 300), (256, 256), (256, 384), (300, 400), (400, 300), (375, 500), (500, 333),
         (257, 1999), (640, 480)]


@pytest.mark.parametrize("resize,out", [(256, 224), (146, 128)])
def test_sizes_against_torchvision(resize, out):
    _check([_image(h, w, seed=h * 7 + w) for h, w in SIZES], resize, out)


def test_identity_resize_is_the_plain_window():
    """A 256-short-side source is not resampled: the output is the window of x / 255, normalised."""
    img = _image(256, 300, seed=1)
    pixels, params = _windows([img], 256, 224)
    got = A.resize_center_crops((pixels, params), dtype=torch.float32).cpu()[0]
    top, left = int(params[0, A.WIN_TOP]), int(params[0, A.WIN_LEFT])
    x = img.permute(2, 0, 1).float()[:, top:top + 224, left:left + 224] / 255
    mean, std = torch.tensor(A.MEAN).view(3, 1, 1), torch.tensor(A.STD).view(3, 1, 1)
    assert torch.equal(got, (x - mean) / std)


def test_column_chunked_source():
    """4000 x 3000: the window spans ~2600 source columns, more than one shared-memory chunk holds."""
    _check([_image(3000, 4000, seed=2), _image(4000, 3000, seed=3)])


def _mixed_batch(n=256, seed=0):
    g = torch.Generator().manual_seed(seed)
    images = []
    for _ in range(n):
        long_side = int(torch.randint(200, 700, (1,), generator=g))
        short = max(1, int(long_side * (0.5 + 0.5 * float(torch.rand(1, generator=g)))))
        h, w = (short, long_side) if float(torch.rand(1, generator=g)) < 0.7 else (long_side, short)
        images.append(_image(h, w, seed=int(torch.randint(0, 1 << 30, (1,), generator=g))))
    return images


def test_seeded_batch_of_mixed_sizes():
    _check(_mixed_batch())


def test_bf16_rounding_bit_identity_and_one_launch():
    pixels, params = _windows(_mixed_batch(32, seed=4), 256, 224)
    f32 = A.resize_center_crops((pixels, params), dtype=torch.float32)
    bf = A.resize_center_crops((pixels, params), dtype=torch.bfloat16)
    assert bf.dtype == torch.bfloat16 and bf.shape == (32, 3, 224, 224)
    assert torch.equal(bf, f32.to(torch.bfloat16))
    assert torch.equal(A.resize_center_crops((pixels, params), dtype=torch.float32), f32)
    assert torch.equal(A.resize_center_crops((pixels, params), dtype=torch.bfloat16), bf)
    torch.cuda.synchronize()
    before = _lib.launches
    A.resize_center_crops((pixels, params))
    torch.cuda.synchronize()
    assert _lib.launches - before == 1


def test_augment_crops_one_crop_per_record():
    torch.manual_seed(7)
    images = [_image(300 + 13 * i, 400 - 11 * i, seed=i) for i in range(12)]
    recs = [A.sample_crop_params(*img.shape[:2], aug="CJ" if i % 2 else "NULL")[None] for i, img in enumerate(images)]
    pixels, params = A.pack_images(images, recs)
    got = A.augment_crops((pixels, params), dtype=torch.float32).cpu()
    assert got.shape == (12, 3, 224, 224)
    worst = max(float((got[i] - A.reference_crop(images[i], params[i])).abs().max()) for i in range(12))
    assert worst <= BOUND, worst


def test_augment_crops_on_two_crop_records_is_augment_two_crop():
    torch.manual_seed(8)
    images = [_image(300 + 13 * i, 400 - 11 * i, seed=i) for i in range(8)]
    recs = [torch.stack([A.sample_crop_params(*img.shape[:2]) for _ in range(2)]) for img in images]
    batch = A.pack_images(images, recs)
    for dtype in (torch.float32, torch.bfloat16):
        one = A.augment_crops(batch, dtype=dtype)
        two = A.augment_two_crop(batch, dtype=dtype)
        assert torch.equal(one.view(8, 6, 224, 224), two)


def _jpeg_split(root, split, sizes, classes=3, seed0=0):
    for c in range(classes):
        os.makedirs(os.path.join(root, split, f"c{c}"), exist_ok=True)
    for i, (h, w) in enumerate(sizes):
        data = torchvision.io.encode_jpeg(_image(h, w, seed=seed0 + i).permute(2, 0, 1).contiguous(), quality=85)
        with open(os.path.join(root, split, f"c{i % classes}", f"{i}.jpg"), "wb") as f:
            f.write(data.numpy().tobytes())


def test_jpeg_folder_end_to_end(tmp_path):
    root = str(tmp_path)
    train_sizes = [(64 + 17 * i, 300 - 9 * i) if i % 2 else (300 - 9 * i, 90 + 11 * i) for i in range(12)]
    val_sizes = [(100, 150), (256, 256), (300, 400), (500, 333), (333, 500), (1200, 900), (257, 640)]
    _jpeg_split(root, "train", train_sizes)
    _jpeg_split(root, "val", val_sizes, seed0=100)

    val = A.ImageFolderEval(os.path.join(root, "val"), train=False)
    loader = torch.utils.data.DataLoader(val, batch_size=3, num_workers=2, pin_memory=True, collate_fn=val.collate_fn)
    seen = []
    for pixels, params, targets, idx in loader:
        assert pixels.is_pinned() and params.is_pinned()
        out = A.resize_center_crops((pixels, params), dtype=torch.float32).cpu()
        for i, k in enumerate(idx.tolist()):
            dec = torchvision.io.decode_image(val.samples[k][0], mode=torchvision.io.ImageReadMode.RGB)
            hwc = dec.permute(1, 2, 0).contiguous()
            ref = A.reference_resize_center_crop(hwc, A.resize_window_params(*hwc.shape[:2]))
            assert float((out[i] - ref).abs().max()) <= BOUND
        assert targets.tolist() == [val.samples[k][1] for k in idx.tolist()]
        seen += idx.tolist()
    assert seen == list(range(len(val)))

    spec = importlib.util.spec_from_file_location("eval_linear_example_gpu", os.path.join(ROOT, "examples",
                                                                                          "eval_linear.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    res = mod.main(["--data-dir", root, "--epochs", "2", "--warmup-epoch", "1", "--total-batch-size", "4",
                    "--num-workers", "0", "--print-freq", "1"])
    assert res["n"] == len(val) and math.isfinite(res["loss"])
    assert all(0.0 <= a <= 100.0 for a in res["acc"]) and res["acc"][1] == 100.0      # top-5 of 3 classes
