"""moco_augment_crops (csrc/augment.cu) on the GPU against torchvision's tensor ops (moco_b200.augment.reference_crop,
fp32 on the CPU) with the same parameters: source sizes from 64 x 64 to 1024 x 768, up- and strong downscaling,
grayscale, all 24 jitter orders, the extreme factors, both flips, two output sizes and one full 256-image batch.
Then bf16 output = fp32 output rounded, run-to-run bit identity, the batch dropping into MoCoStep's input path, and
the JPEG folder end to end through the loader."""
import itertools
import os

import pytest
import torch
import torchvision

from moco_b200 import _lib
from moco_b200 import augment as A

pytestmark = pytest.mark.gpu
BOUND = 1e-4          # max |kernel - torchvision| in normalised units


def _image(h, w, seed):
    g = torch.Generator().manual_seed(seed)
    base = torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.int32)
    # smooth structure plus noise, and a few saturated / grey pixels (hue's degenerate cases)
    yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    smooth = torch.stack([(yy * 255) // max(h - 1, 1), (xx * 255) // max(w - 1, 1), ((yy + xx) * 7) % 256], -1)
    img = ((base + 3 * smooth) // 4).to(torch.uint8)
    img[: h // 8, : w // 8] = 128
    img[-2:, -2:] = 255
    return img.contiguous()


def _rec(h, w, top, left, ch, cw, flags=0, order=(0, 1, 2, 3), b=1.0, c=1.0, s=1.0, hue=0.0):
    o = sum(op << (2 * k) for k, op in enumerate(order))
    bits = torch.tensor([b, c, s, hue], dtype=torch.float32).view(torch.int32).tolist()
    return torch.tensor([0, 0, h, w, top, left, ch, cw, flags, o] + bits, dtype=torch.int32)


def _pack(images, recs_per_image):
    """[(hwc)], [[rec, rec]] -> (pixels, params) as ImageFolderTwoCrop.collate_fn packs them."""
    items = [(img, torch.stack(recs), 0) for img, recs in zip(images, recs_per_image)]
    pixels, params, _ = A.ImageFolderTwoCrop.collate_fn(items)
    return pixels, params


def _check(images, recs_per_image, out_size=224):
    pixels, params = _pack(images, recs_per_image)
    got = A.augment_two_crop((pixels, params), out_size=out_size, dtype=torch.float32).cpu()
    oh, ow = (out_size, out_size) if isinstance(out_size, int) else out_size
    got = got.view(-1, 3, oh, ow)
    worst = 0.0
    for i in range(got.shape[0]):
        ref = A.reference_crop(images[i // 2], params[i], out_size)
        worst = max(worst, float((got[i] - ref).abs().max()))
    print(f"max |diff| = {worst:.3g}")
    assert worst <= BOUND, worst
    return worst


J = _lib.AUG_JITTER
G = _lib.AUG_GRAY
F = _lib.AUG_FLIP


@pytest.mark.parametrize("hw", [(64, 64), (768, 1024), (1024, 768), (97, 131), (375, 500), (500, 375)])
@pytest.mark.parametrize("out_size", [224, (64, 48)])
def test_sizes_scales_and_flips(hw, out_size):
    h, w = hw
    img = _image(h, w, seed=h * 7 + w)
    recs = [
        [_rec(h, w, 0, 0, h, w), _rec(h, w, 0, 0, h, w, F)],                                   # whole image, both flips
        [_rec(h, w, h // 5, w // 7, max(1, h // 9), max(1, w // 11), F | J, (3, 1, 0, 2), 1.4, 0.6, 1.4, 0.4),  # upscale
         _rec(h, w, 1, 2, h - 3, w - 2, J, (2, 0, 3, 1), 0.6, 1.4, 0.6, -0.4)],               # downscale
        [_rec(h, w, h // 3, 0, h - h // 3, w, G | J, (1, 3, 2, 0), 1.1, 1.4, 0.6, 0.0),
         _rec(h, w, 0, w // 2, max(1, h // 2), w - w // 2, G | F)],
    ]
    _check([img] * len(recs), recs, out_size)


def test_all_24_jitter_orders():
    h, w = 181, 243
    img = _image(h, w, seed=5)
    recs = []
    for k, order in enumerate(itertools.permutations(range(4))):
        factors = [(0.6, 1.4, 0.6, 0.4), (1.4, 0.6, 1.4, -0.4), (0.9, 1.2, 0.8, 0.1)][k % 3]
        recs.append(_rec(h, w, k, 2 * k, h - 2 * k, w - 3 * k, J | (F if k % 2 else 0) | (G if k % 5 == 0 else 0),
                         order, *factors))
    _check([img] * 12, [recs[2 * i:2 * i + 2] for i in range(12)])


def test_full_batch_of_drawn_parameters():
    """256 images of 500 x 375 (landscape and portrait), 512 crops drawn by the sampler as the loader draws them."""
    torch.manual_seed(11)
    images, recs = [], []
    for n in range(256):
        h, w = (375, 500) if n % 3 else (500, 375)
        images.append(_image(h, w, seed=1000 + n))
        recs.append([A.sample_crop_params(h, w, aug="CJ") for _ in range(2)])
    _check(images, recs)


def _batch(n=16, seed=0):
    torch.manual_seed(seed)
    images = [_image(300 + 13 * i, 400 - 11 * i, seed=i) for i in range(n)]
    recs = [[A.sample_crop_params(*img.shape[:2]) for _ in range(2)] for img in images]
    return _pack(images, recs)


def test_bf16_is_the_rounded_fp32_output_and_runs_are_bit_identical():
    batch = _batch()
    f32 = A.augment_two_crop(batch, dtype=torch.float32)
    bf = A.augment_two_crop(batch, dtype=torch.bfloat16)
    assert bf.dtype == torch.bfloat16 and bf.shape == (16, 6, 224, 224)
    assert torch.equal(bf, f32.to(torch.bfloat16))
    assert torch.equal(A.augment_two_crop(batch, dtype=torch.float32), f32)
    assert torch.equal(A.augment_two_crop(batch, dtype=torch.bfloat16), bf)


def test_batch_drops_into_the_step_input_path():
    """MoCoStep(channels_last=True) on the bf16 batch and on that batch .float(): identical loss, prob and weights."""
    from moco_b200 import encoders
    from moco_b200.NCE import MemoryMoCo
    from moco_b200.train_step import MoCoStep
    inputs = A.augment_two_crop(_batch(), dtype=torch.bfloat16)
    results = []
    for x in (inputs, inputs.float()):
        torch.manual_seed(0)
        model = encoders.resnet18(low_dim=128).cuda().to(memory_format=torch.channels_last)
        ema = encoders.resnet18(low_dim=128).cuda().to(memory_format=torch.channels_last)
        ema.load_state_dict(model.state_dict())
        contrast = MemoryMoCo(128, 1024, 0.07).cuda()
        opt = torch.optim.SGD(model.parameters(), lr=0.003, momentum=0.9, weight_decay=1e-4)
        step = MoCoStep(model, ema, contrast, opt, channels_last=True)
        x1, x2 = torch.split(x, [3, 3], dim=1)
        loss, prob = step(x1, x2, 1)
        torch.cuda.synchronize()
        results.append((loss.detach().clone(), prob.detach().clone(),
                        [p.detach().clone() for p in model.parameters()]))
    (l0, p0, w0), (l1, p1, w1) = results
    assert torch.isfinite(l0) and torch.equal(l0, l1) and torch.equal(p0, p1)
    assert all(torch.equal(a, b) for a, b in zip(w0, w1))


def test_jpeg_folder_end_to_end(tmp_path):
    sizes = [(64, 80), (97, 61), (240, 320), (333, 250), (50, 500), (768, 1024)]
    for c in range(2):
        os.makedirs(tmp_path / "train" / f"c{c}")
    for i, (h, w) in enumerate(sizes):
        data = torchvision.io.encode_jpeg(_image(h, w, seed=i).permute(2, 0, 1).contiguous(), quality=85)
        (tmp_path / "train" / f"c{i % 2}" / f"{i}.jpg").write_bytes(data.numpy().tobytes())
    ds = A.ImageFolderTwoCrop(str(tmp_path / "train"), scale=(0.08, 1.0), aug="CJ")
    loader = torch.utils.data.DataLoader(ds, batch_size=3, num_workers=2, pin_memory=True, drop_last=True,
                                         collate_fn=A.ImageFolderTwoCrop.collate_fn,
                                         worker_init_fn=lambda w: torch.manual_seed(77 + w))
    seen = 0
    for pixels, params, _ in loader:
        assert pixels.is_pinned() and params.is_pinned()
        out = A.augment_two_crop((pixels, params), dtype=torch.float32).cpu().view(-1, 3, 224, 224)
        for i in range(out.shape[0]):
            r = params[i].tolist()
            off, h, w = r[A.OFF_LO], r[A.SRC_H], r[A.SRC_W]
            img = pixels[off:off + h * w * 3].view(h, w, 3)
            assert float((out[i] - A.reference_crop(img, params[i])).abs().max()) <= BOUND
            seen += 1
    assert seen == 12
