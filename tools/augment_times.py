"""Cost of the two-crop augmentation on the GPU (moco_augment_crops) and of the loader that feeds it.

  - Kernel: CUDA events around `--iters` warm calls of moco_augment_crops on one 256-image batch (512 crops, bf16
    224 x 224 output) already on the device, sources of ImageNet-like sizes (seeded), parameters drawn by the
    sampler.  Also the max |diff| of that batch against torchvision's tensor ops (moco_b200.augment.reference_crop).
  - Loader: images per second out of a DataLoader with os.cpu_count() workers over a seeded synthetic JPEG folder
    written under the output directory, decode-only (ImageFolderTwoCrop) against the reference's PIL two-crop
    transform (train.py:106-114 applied twice per image as moco/dataset.py does).  The first epoch warms the workers
    and the page cache; the second is timed.
Writes one JSON object with the card's name, power limit and the host's CPU count.

    python tools/augment_times.py --out DIR [--images 2048] [--iters 50]

DIR (default: a directory under the system's temporary directory) receives the JSON and the JPEG folder.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, watts = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit_w": float(watts)}
    except Exception:
        return {}


def imagenet_like_size(g):
    """(h, w) around ImageNet's typical 500 x 375 / 375 x 500, with some larger and smaller images."""
    import torch
    long_side = int(torch.randint(300, 640, (1,), generator=g))
    short = int(long_side * (0.6 + 0.15 * float(torch.rand(1, generator=g))))
    return (short, long_side) if float(torch.rand(1, generator=g)) < 0.75 else (long_side, short)


def image(h, w, g):
    import torch
    yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    base = torch.stack([(yy * 255) // h, (xx * 255) // w, ((yy + 2 * xx) * 3) % 256], -1)
    noise = torch.randint(0, 64, (h, w, 3), generator=g)
    return ((base * 3 + noise * 4) // 4).clamp(0, 255).to(torch.uint8).contiguous()


def kernel_times(iters):
    import torch
    from moco_b200 import _lib
    from moco_b200 import augment as A
    g = torch.Generator().manual_seed(0)
    torch.manual_seed(0)
    items = []
    for _ in range(256):
        h, w = imagenet_like_size(g)
        items.append((image(h, w, g), torch.stack([A.sample_crop_params(h, w) for _ in range(2)]), 0))
    pixels, params, _ = A.ImageFolderTwoCrop.collate_fn(items)
    dev = torch.device("cuda", 0)
    pix, prm = pixels.to(dev), params.to(dev)
    out = torch.empty(512, 3, 224, 224, dtype=torch.bfloat16, device=dev)
    means = torch.empty(512, dtype=torch.float32, device=dev)
    import ctypes
    norm = (ctypes.c_float * 6)(*A.MEAN, *A.STD)
    lib = _lib.load()

    def call(dst, dtype):
        _lib.check(lib.moco_augment_crops(pix.data_ptr(), pix.numel(), prm.data_ptr(), 512, 224, 224, norm,
                                          dst.data_ptr(), dtype, means.data_ptr(), _lib.cur_stream()), "augment")

    for _ in range(5):
        call(out, _lib.MOCO_BF16)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record()
    for _ in range(iters):
        call(out, _lib.MOCO_BF16)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1) / iters
    # the host-to-device copy of the batch from pinned memory, for comparison with the fp32 crops it replaces
    pinned = pixels.pin_memory()
    torch.cuda.synchronize()
    ev0.record()
    for _ in range(iters):
        pix.copy_(pinned, non_blocking=True)
    ev1.record()
    torch.cuda.synchronize()
    h2d_ms = ev0.elapsed_time(ev1) / iters
    f32 = torch.empty(512, 3, 224, 224, dtype=torch.float32, device=dev)
    call(f32, _lib.MOCO_F32)
    got = f32.cpu()
    worst = 0.0
    for i in range(0, 512, 4):                    # every other image's first crop and a quarter of the batch
        worst = max(worst, float((got[i] - A.reference_crop(items[i // 2][0], params[i])).abs().max()))
    return {"batch_images": 256, "crops": 512, "out": [224, 224], "dtype": "bf16", "iters": iters,
            "kernel_ms_per_batch": round(ms, 4), "pixels_bytes": int(pixels.numel()),
            "h2d_pinned_ms_per_batch": round(h2d_ms, 4),
            "max_abs_diff_vs_torchvision_fp32_128_crops": worst}


def write_folder(root, n):
    import torch
    import torchvision
    g = torch.Generator().manual_seed(1)
    for c in range(8):
        os.makedirs(os.path.join(root, "train", f"class{c}"), exist_ok=True)
    for i in range(n):
        path = os.path.join(root, "train", f"class{i % 8}", f"{i:05d}.jpg")
        if os.path.exists(path):
            continue
        h, w = imagenet_like_size(g)
        data = torchvision.io.encode_jpeg(image(h, w, g).permute(2, 0, 1).contiguous(), quality=90)
        with open(path, "wb") as f:
            f.write(data.numpy().tobytes())


class _ReferenceTwoCrop:
    """moco/dataset.py's ImageFolderInstance(two_crop=True) with train.py's CJ transform on PIL images."""

    def __init__(self, root):
        import torchvision
        from torchvision import transforms as T
        from moco_b200 import augment as A
        self.ds = torchvision.datasets.ImageFolder(root)
        self.t = T.Compose([T.RandomResizedCrop(224, scale=(0.08, 1.0)), T.RandomGrayscale(p=0.2),
                            T.ColorJitter(0.4, 0.4, 0.4, 0.4), T.RandomHorizontalFlip(), T.ToTensor(),
                            T.Normalize(mean=A.MEAN, std=A.STD)])

    def __len__(self):
        return len(self.ds)

    def __getitem__(self, i):
        import torch
        path, target = self.ds.samples[i]
        img = self.ds.loader(path)
        return torch.cat([self.t(img), self.t(img)], dim=0), target


def loader_rate(ds, workers, batch, collate=None):
    import torch
    kw = {"collate_fn": collate} if collate else {}
    loader = torch.utils.data.DataLoader(ds, batch_size=batch, shuffle=False, num_workers=workers, pin_memory=True,
                                         drop_last=True, persistent_workers=True, **kw)
    for _ in loader:                               # warm-up epoch
        pass
    t0 = time.perf_counter()
    n = 0
    for b in loader:
        n += b[0].shape[0] if collate is None else b[1].shape[0] // 2
    dt = time.perf_counter() - t0
    del loader
    return {"images": n, "seconds": round(dt, 3), "img_per_s": round(n / dt, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "moco_augment_times"))
    ap.add_argument("--images", type=int, default=2048)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--batch", type=int, default=128)
    args = ap.parse_args()
    import torch
    from moco_b200.augment import ImageFolderTwoCrop
    os.makedirs(args.out, exist_ok=True)
    res = {"card": card(), "cpu_count": os.cpu_count(), "torch": torch.__version__}
    res["kernel"] = kernel_times(args.iters)
    res["kernel"]["share_of_60ms_step"] = round(res["kernel"]["kernel_ms_per_batch"] / 60.0, 5)
    print(json.dumps(res), flush=True)
    data = os.path.join(args.out, "augment_data")
    write_folder(data, args.images)
    workers = os.cpu_count() or 1
    res["loader"] = {"workers": workers, "batch": args.batch, "folder_images": args.images,
                     "decode_only": loader_rate(ImageFolderTwoCrop(os.path.join(data, "train")), workers, args.batch,
                                                ImageFolderTwoCrop.collate_fn),
                     "reference_pil_transform": loader_rate(_ReferenceTwoCrop(os.path.join(data, "train")), workers,
                                                            args.batch)}
    print(json.dumps(res), flush=True)
    with open(os.path.join(args.out, "augment_times_h100.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
