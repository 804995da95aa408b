"""Time of the pre-training recipe (examples/train_moco.py --data-dir) on one GPU: ResNet-50, 256 images per step,
K = 65536, over a seeded folder of ImageNet-sized JPEGs (tools/augment_times.py's generator).  In one process:

  (a) GPU side.  Recipe steps (moco_augment_crops + MoCoStep + the two device-side loss / prob sums) fed from a
      cycle of pre-decoded, pinned batches, so that no decoding is on the path.  Two arms, alternated over
      ``--rounds`` rounds of ``--steps`` steps: the packed pixels copied on the compute stream (augment_two_crop on
      the pinned batch), and prefetched on a copy stream (moco_b200.augment.prefetch_pixels).  Each round is timed
      by the host clock between two device synchronisations.  Also the host-to-device copy of one batch's pixels,
      timed by events on the copy stream with nothing else running.
  (b) Whole loop.  examples/train_moco.py's recipe over the folder for two epochs with os.cpu_count() workers;
      images per second and mean data wait per step of the second epoch.  This is bound by CPU decoding.
  (c) Reference point.  MoCoStep on one synthetic device-resident batch, no augmentation and no copy.
The JPEG folder (``--data``) and the recipe's checkpoints go to the system's temporary directory.  Writes
DIR/pretrain_epoch_h100.json with the card's name, power limit and SM clocks, and the host's CPU count.

    python tools/pretrain_epoch_times.py --out DIR [--images 2560] [--rounds 4] [--steps 20]
"""
from __future__ import annotations

import argparse
import importlib.util
import itertools
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from augment_times import write_folder  # noqa: E402  (seeded ImageNet-sized JPEGs)
from eval_data_times import card, sm_clock  # noqa: E402

BATCH, K = 256, 65536


def _models(dev):
    import torch
    from moco_b200 import encoders
    from moco_b200.NCE import MemoryMoCo
    from moco_b200.train_step import MoCoStep
    from moco_b200.util import moment_update
    torch.manual_seed(0)
    model = encoders.resnet50(low_dim=128).to(dev).to(memory_format=torch.channels_last)
    ema = encoders.resnet50(low_dim=128).to(dev).to(memory_format=torch.channels_last)
    moment_update(model, ema, 0)
    contrast = MemoryMoCo(128, K, 0.07).to(dev)
    opt = torch.optim.SGD(model.parameters(), lr=BATCH / 256 * 0.1, momentum=0.9, weight_decay=1e-4)
    return MoCoStep(model, ema, contrast, opt, channels_last=True)


def pinned_batches(folder, n):
    import torch
    from moco_b200.augment import ImageFolderTwoCrop
    ds = ImageFolderTwoCrop(os.path.join(folder, "train"))
    torch.manual_seed(1)
    out = []
    for b in range(n):
        pixels, params, targets = ImageFolderTwoCrop.collate_fn([ds[i] for i in range(b * BATCH, (b + 1) * BATCH)])
        out.append((pixels.pin_memory(), params, targets))
    return out


def gpu_side(folder, rounds, steps, dev):
    import torch
    from moco_b200.augment import augment_two_crop, prefetch_pixels
    batches = pinned_batches(folder, 4)
    step = _models(dev)
    sums = torch.zeros(2, device=dev)

    def run(source, n):
        for batch in itertools.islice(source, n):
            x1, x2 = torch.split(augment_two_crop(batch), [3, 3], dim=1)
            loss, prob = step(x1, x2, 1)
            sums[0].add_(loss.detach(), alpha=BATCH)
            sums[1].add_(prob.detach(), alpha=BATCH)

    arms = {"copy_on_compute_stream": lambda: itertools.cycle(batches),
            "prefetch_on_copy_stream": lambda: prefetch_pixels(itertools.cycle(batches), dev)}
    for make in arms.values():
        run(make(), 3)                                                      # warm-up, both arms
    times = {name: [] for name in arms}
    clocks = []
    for _ in range(rounds):
        for name, make in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(make(), steps)
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) / steps * 1e3)
            clocks.append(sm_clock())
    res = {name: {"ms_per_step": [round(t, 3) for t in ts], "mean_ms": round(statistics.mean(ts), 3),
                  "min_ms": round(min(ts), 3), "max_ms": round(max(ts), 3),
                  "img_per_s_mean": round(BATCH / statistics.mean(ts) * 1e3, 1)} for name, ts in times.items()}

    copy = torch.cuda.Stream(dev)
    dst = torch.empty_like(batches[0][0], device=dev)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    h2d = []
    torch.cuda.synchronize()
    for i in range(20):
        src = batches[i % len(batches)][0]
        if dst.numel() != src.numel():
            dst = torch.empty_like(src, device=dev)
        with torch.cuda.stream(copy):
            ev0.record(copy)
            dst.copy_(src, non_blocking=True)
            ev1.record(copy)
        ev1.synchronize()
        h2d.append(ev0.elapsed_time(ev1))
    mb = statistics.mean(b[0].numel() for b in batches) / 1e6
    res.update({"rounds": rounds, "steps_per_round": steps, "sm_mhz_after_each_window": clocks,
                "pixels_mb_per_batch_mean": round(mb, 1),
                "h2d_ms_per_batch_copy_stream": round(statistics.median(h2d), 3),
                "h2d_gb_per_s": round(mb / statistics.median(h2d), 2),
                "prefetch_gain_ms_per_step": round(res["copy_on_compute_stream"]["mean_ms"]
                                                   - res["prefetch_on_copy_stream"]["mean_ms"], 3)})
    del step, batches
    return res


def whole_loop(folder, workers):
    spec = importlib.util.spec_from_file_location("train_moco_timing", os.path.join(ROOT, "examples", "train_moco.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    with tempfile.TemporaryDirectory(prefix="moco_pretrain_ckpt_") as ckpt_dir:
        r = mod.main(["--data-dir", folder, "--batch-size", str(BATCH), "--nce-k", str(K), "--epochs", "2",
                      "--warmup-epoch", "1", "--num-workers", str(workers), "--print-freq", "1000000",
                      "--save-freq", "1000000", "--output-dir", ckpt_dir])
    return {"workers": workers, "cpu_count": os.cpu_count(), "steps": r["steps"], "epoch_seconds": round(r["seconds"], 3),
            "img_per_s": round(r["steps"] * BATCH / r["seconds"], 1),
            "data_wait_ms_per_step": round(r["data_wait_seconds"] / r["steps"] * 1e3, 3), "loss": r["loss"]}


def synthetic(steps, dev):
    import torch
    step = _models(dev)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(BATCH, 6, 224, 224, device=dev, generator=g)
    x1, x2 = torch.split(x, [3, 3], dim=1)
    for _ in range(3):
        step(x1, x2, 1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        step(x1, x2, 1)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) / steps * 1e3
    return {"ms_per_step": round(ms, 3), "img_per_s": round(BATCH / ms * 1e3, 1), "steps": steps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "moco_pretrain_epoch_times"))
    ap.add_argument("--data", default=os.path.join(tempfile.gettempdir(), "moco_pretrain_jpegs"))
    ap.add_argument("--images", type=int, default=2560)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("pretrain_epoch_times.py measures the GPU; there is no CPU fallback")
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    os.makedirs(args.out, exist_ok=True)
    write_folder(args.data, args.images)
    res = {"card": card(), "cpu_count": os.cpu_count(), "torch": torch.__version__, "batch": BATCH, "K": K,
           "arch": "resnet50", "folder_images": args.images}
    res["a_gpu_side"] = gpu_side(args.data, args.rounds, args.steps, dev)
    print(json.dumps(res), flush=True)
    torch.cuda.empty_cache()
    res["c_synthetic_step"] = synthetic(args.steps, dev)
    torch.cuda.empty_cache()
    res["b_whole_loop"] = whole_loop(args.data, os.cpu_count() or 1)
    res["sm_mhz_at_end"] = sm_clock()
    print(json.dumps(res), flush=True)
    with open(os.path.join(args.out, "pretrain_epoch_h100.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
