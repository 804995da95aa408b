"""Cost of the linear evaluation's validation transform on the GPU (moco_resize_center_crops) and of the loader that
feeds it, beside the frozen probe step it feeds.

  - Kernel: CUDA events around `--iters` warm calls (three windows) of moco_resize_center_crops on one seeded 256-image batch (bf16
    224 x 224 output of Resize(256) -> CenterCrop(224)) already on the device; sources mostly 500 x 375, 375 x 500 and
    500 x 333 with a few large ones.  Reports the uint8 bytes of the batch, the bytes under the windows' source
    footprint (what the kernel has to read), the bytes written and the achieved bandwidth, and the max |diff| of part
    of the batch against torchvision's tensor ops (moco_b200.augment.reference_resize_center_crop).
  - Probe step: a frozen ResNet-50's `model(x, 6)` under bf16 autocast + the linear classifier's forward, loss,
    backward and SGD step at 256 images, timed the same way, and the transform's share of it.
  - Loader: images per second out of a DataLoader with os.cpu_count() workers over a seeded synthetic JPEG folder,
    decode-only ImageFolderEval val workers against the reference's PIL validation transform (eval.py:111-116).  The
    first epoch warms the workers and the page cache; the second is timed.
Writes one JSON object with the card's name and power limit, the SM clock sampled right after each timed window, and
the host's CPU count.

    python tools/eval_data_times.py --out DIR [--images 2048] [--iters 500]
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
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from augment_times import image  # noqa: E402  (the seeded synthetic image of the augmentation timing)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, watts, sm, sm_max = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit_w": float(watts), "sm_clock_mhz": float(sm), "max_sm_clock_mhz": float(sm_max)}
    except Exception:
        return {}


def sm_clock():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return float(out)
    except Exception:
        return None


def val_size(g):
    """Mostly ImageNet's 500 x 375 / 375 x 500 / 500 x 333, 2 % large (up to 2048 px)."""
    import torch
    r = float(torch.rand(1, generator=g))
    if r < 0.02:
        long_side = int(torch.randint(1200, 2049, (1,), generator=g))
        return (long_side * 3 // 4, long_side)
    if r < 0.9:
        return [(375, 500), (500, 375), (333, 500), (500, 333)][int(torch.randint(0, 4, (1,), generator=g))]
    return (int(torch.randint(200, 500, (1,), generator=g)), int(torch.randint(200, 500, (1,), generator=g)))


def footprint(in_size, resized, origin, n):
    """Source rows (or columns) the window's taps touch: [lo of the first output, hi of the last)."""
    scale = in_size / resized
    support = max(scale, 1.0)
    lo = max(int(scale * (origin + 0.5) - support + 0.5), 0)
    hi = min(int(scale * (origin + n - 0.5) + support + 0.5), in_size)
    return hi - lo


def timed(fn, iters, warmup=5):
    import torch
    for _ in range(warmup):
        fn()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record()
    for _ in range(iters):
        fn()
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / iters


def kernel_times(iters):
    import ctypes
    import torch
    from moco_b200 import _lib
    from moco_b200 import augment as A
    g = torch.Generator().manual_seed(0)
    images = [image(*val_size(g), g) for _ in range(256)]
    recs = [A.resize_window_params(img.shape[0], img.shape[1])[None] for img in images]
    pixels, params = A.pack_images(images, recs)
    dev = torch.device("cuda", 0)
    pix, prm = pixels.to(dev), params.to(dev)
    out = torch.empty(256, 3, 224, 224, dtype=torch.bfloat16, device=dev)
    norm = (ctypes.c_float * 6)(*A.MEAN, *A.STD)
    lib = _lib.load()

    def call(dst, dtype):
        _lib.check(lib.moco_resize_center_crops(pix.data_ptr(), pix.numel(), prm.data_ptr(), 256, 224, 224, norm,
                                                dst.data_ptr(), dtype, _lib.cur_stream()), "resize")

    windows = []
    for _ in range(3):
        windows.append(round(timed(lambda: call(out, _lib.MOCO_BF16), iters), 4))
        windows.append(sm_clock())
    ms = sorted(windows[0::2])[1]                 # the median window
    read = sum(footprint(r[2], r[4], r[6], 224) * footprint(r[3], r[5], r[7], 224) * 3 for r in params.tolist())
    written = out.numel() * out.element_size()
    f32 = torch.empty(256, 3, 224, 224, dtype=torch.float32, device=dev)
    call(f32, _lib.MOCO_F32)
    got = f32.cpu()
    worst = max(float((got[i] - A.reference_resize_center_crop(images[i], params[i])).abs().max())
                for i in range(0, 256, 4))
    large = sum(1 for img in images if max(img.shape[:2]) > 1000)
    return {"batch_images": 256, "large_sources": large, "out": [224, 224], "dtype": "bf16", "iters": iters,
            "kernel_ms_per_batch": round(ms, 4), "kernel_ms_windows_and_sm_mhz_after": windows,
            "pixels_bytes": int(pixels.numel()),
            "window_footprint_bytes": int(read), "bytes_written": int(written),
            "gb_per_s_footprint_plus_written": round((read + written) / ms / 1e6, 1),
            "max_abs_diff_vs_torchvision_fp32_64_images": worst}


def probe_step_ms(iters):
    import torch
    from moco_b200.encoders import resnet50
    from moco_b200.linear_eval import LinearClassifierResNet
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    model = resnet50().to(dev).to(memory_format=torch.channels_last)
    model.freeze()
    clf = LinearClassifierResNet(6, 1000).to(dev)
    opt = torch.optim.SGD(clf.parameters(), lr=30.0, momentum=0.9)
    crit = torch.nn.CrossEntropyLoss()
    x = torch.randn(256, 3, 224, 224, device=dev).bfloat16()
    y = torch.randint(0, 1000, (256,), device=dev)

    def step():
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            feat = model(x, 6).float()
        loss = crit(clf(feat), y)
        opt.zero_grad()
        loss.backward()
        opt.step()

    ms = timed(step, iters, warmup=5)
    return ms, sm_clock()


def write_folder(root, n):
    import torch
    import torchvision
    g = torch.Generator().manual_seed(1)
    for c in range(8):
        os.makedirs(os.path.join(root, "val", f"class{c}"), exist_ok=True)
    for i in range(n):
        path = os.path.join(root, "val", f"class{i % 8}", f"{i:05d}.jpg")
        h, w = val_size(g)
        img = image(h, w, g)
        if os.path.exists(path):
            continue
        data = torchvision.io.encode_jpeg(img.permute(2, 0, 1).contiguous(), quality=90)
        with open(path, "wb") as f:
            f.write(data.numpy().tobytes())


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
        n += b[1].shape[0]
    dt = time.perf_counter() - t0
    del loader
    return {"images": n, "seconds": round(dt, 3), "img_per_s": round(n / dt, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "moco_eval_data_times"))
    ap.add_argument("--images", type=int, default=2048)
    ap.add_argument("--iters", type=int, default=500)
    ap.add_argument("--batch", type=int, default=128)
    args = ap.parse_args()
    import torch
    import torchvision
    from torchvision import transforms as T
    from moco_b200 import augment as A
    os.makedirs(args.out, exist_ok=True)
    res = {"card": card(), "cpu_count": os.cpu_count(), "torch": torch.__version__}
    res["kernel"] = kernel_times(args.iters)
    ms, mhz = probe_step_ms(max(args.iters // 5, 20))
    res["probe_step_ms_256"] = round(ms, 3)
    res["probe_step_sm_mhz_after"] = mhz
    share = res["kernel"]["kernel_ms_per_batch"] / res["probe_step_ms_256"]
    res["transform_share_of_probe_step"] = round(share, 5)
    res["target_below_10_percent_met"] = share < 0.10
    print(json.dumps(res), flush=True)
    data = os.path.join(args.out, "eval_data")
    write_folder(data, args.images)
    workers = os.cpu_count() or 1
    val = os.path.join(data, "val")
    ds = A.ImageFolderEval(val, train=False)
    ref = torchvision.datasets.ImageFolder(val, T.Compose([T.Resize(256), T.CenterCrop(224), T.ToTensor(),
                                                           T.Normalize(mean=A.MEAN, std=A.STD)]))
    res["loader"] = {"workers": workers, "batch": args.batch, "folder_images": args.images,
                     "decode_only": loader_rate(ds, workers, args.batch, ds.collate_fn),
                     "reference_pil_transform": loader_rate(ref, workers, args.batch)}
    print(json.dumps(res), flush=True)
    with open(os.path.join(args.out, "eval_data_times_h100.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
