"""MoCo v2's augmentation and MLP head on one GPU, in one process:

  (a) The device time of one seeded 256-image batch (512 crops of ImageNet-sized sources, bf16 224 x 224) through
      moco_augment_crops with CJ records and through moco_augment_crops_blur with V2 records, the two alternated over
      ``--rounds`` rounds of ``--iters`` calls, each window timed by CUDA events.
  (b) In a separate profiled pass, each augmentation kernel's device time per V2 batch (torch.profiler), the blur
      apply kernel's among them.
  (c) Max |diff| of the V2 batch (fp32) against torchvision's tensor transform (augment.reference_crop) over a quarter
      of its crops.
  (d) Registers, shared memory and spills of the augmentation kernels, from nvcc -Xptxas -v on csrc/augment.cu.
  (e) The recipe's step (augment_two_crop + MoCoStep, ResNet-50, K = 65536) on pre-decoded pinned V2 batches, with
      and without the MLP head, alternated over ``--rounds`` rounds of ``--steps`` steps, host clock between device
      synchronisations.
Writes DIR/augment_v2_times_h100.json with the card's name, power limit and SM clocks.

    python tools/augment_v2_times.py --out DIR [--rounds 5] [--iters 30] [--steps 10]
"""
from __future__ import annotations

import argparse
import ctypes
import itertools
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from augment_times import image, imagenet_like_size  # noqa: E402
from eval_data_times import card, sm_clock  # noqa: E402

BATCH, K = 256, 65536


def batch(aug, seed):
    """A pinned (pixels, params, targets) batch of 256 seeded ImageNet-sized images, two crops each."""
    import torch
    from moco_b200 import augment as A
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    items = []
    for _ in range(BATCH):
        h, w = imagenet_like_size(g)
        items.append((image(h, w, g), torch.stack([A.sample_crop_params(h, w, (0.2, 1.0), aug) for _ in range(2)]),
                      0))
    pixels, params, targets = A.ImageFolderTwoCrop.collate_fn(items)
    return (pixels.pin_memory(), params, targets), items


def augment_times(rounds, iters, dev):
    import torch
    from moco_b200 import _lib
    from moco_b200 import augment as A
    lib = _lib.load()
    norm = (ctypes.c_float * 6)(*A.MEAN, *A.STD)
    out = torch.empty(2 * BATCH, 3, 224, 224, dtype=torch.bfloat16, device=dev)
    means = torch.empty(2 * BATCH, dtype=torch.float32, device=dev)
    arms = {}
    for aug in ("CJ", "V2"):
        (pixels, params, _), items = batch(aug, 0)                  # the same images and crop boxes under both
        pix, prm = pixels.to(dev), params.to(dev)

        def call(dst, dtype, pix=pix, prm=prm, aug=aug):
            if aug == "V2":
                _lib.check(lib.moco_augment_crops_blur(pix.data_ptr(), pix.numel(), prm.data_ptr(), 2 * BATCH, 224,
                                                       224, A.BLUR_KSIZE, norm, dst.data_ptr(), dtype,
                                                       means.data_ptr(), _lib.cur_stream()), "augment V2")
            else:
                _lib.check(lib.moco_augment_crops(pix.data_ptr(), pix.numel(), prm.data_ptr(), 2 * BATCH, 224, 224,
                                                  norm, dst.data_ptr(), dtype, means.data_ptr(), _lib.cur_stream()),
                           "augment CJ")
        arms[aug] = (call, params, items)
    for call, _, _ in arms.values():
        for _ in range(5):
            call(out, _lib.MOCO_BF16)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = {aug: [] for aug in arms}
    for _ in range(rounds):
        for aug, (call, _, _) in arms.items():
            torch.cuda.synchronize()
            ev0.record()
            for _ in range(iters):
                call(out, _lib.MOCO_BF16)
            ev1.record()
            torch.cuda.synchronize()
            times[aug].append(ev0.elapsed_time(ev1) / iters)
    res = {aug: {"ms_per_batch": [round(t, 4) for t in ts], "median_ms": round(statistics.median(ts), 4)}
           for aug, ts in times.items()}
    v2_params = arms["V2"][1]
    res["v2_over_cj"] = round(res["V2"]["median_ms"] / res["CJ"]["median_ms"], 3)
    res["v2_blurred_crops"] = int(v2_params[:, A.BLUR].sum())
    res["v2_jittered_crops"] = int((v2_params[:, A.FLAGS] & _lib.AUG_JITTER != 0).sum())
    res["cj_jittered_crops"] = int((arms["CJ"][1][:, A.FLAGS] & _lib.AUG_JITTER != 0).sum())

    # (b) per-kernel device time, in a profiled pass of its own
    from torch.profiler import ProfilerActivity, profile
    n_prof = 10
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n_prof):
            arms["V2"][0](out, _lib.MOCO_BF16)
        torch.cuda.synchronize()
    kernels = {}
    for evt in prof.key_averages():
        m = re.search(r"(aug_\w+_kernel)", evt.key)
        if m:
            kernels[m.group(1)] = round(evt.device_time_total / n_prof / 1e3, 4)
    res["v2_kernel_ms_per_batch"] = kernels

    # (c) the V2 batch against torchvision's tensor transform
    f32 = torch.empty(2 * BATCH, 3, 224, 224, dtype=torch.float32, device=dev)
    arms["V2"][0](f32, _lib.MOCO_F32)
    got = f32.cpu()
    items = arms["V2"][2]
    worst = 0.0
    for i in range(0, 2 * BATCH, 4):
        worst = max(worst, float((got[i] - A.reference_crop(items[i // 2][0], v2_params[i])).abs().max()))
    res["v2_max_abs_diff_vs_torchvision_fp32_128_crops"] = worst
    res.update({"batch_images": BATCH, "crops": 2 * BATCH, "out": [224, 224], "dtype": "bf16", "rounds": rounds,
                "iters_per_round": iters})
    return res


def ptxas():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler",
                            "-fPIC", "-Xptxas", "-v", "-c", os.path.join(ROOT, "moco_b200", "csrc", "augment.cu"),
                            "-o", os.path.join(tmp, "augment.o")], capture_output=True, text=True)
    res, name = {}, None
    for line in (r.stdout + r.stderr).splitlines():
        m = re.search(r"Compiling entry function '\w*?(\d+)(aug_\w+_kernel|resize_window_kernel)", line)
        if m:
            name = m.group(2)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            res.setdefault(name, {})["spill_bytes"] = int(m.group(1)) + int(m.group(2))
        m = re.search(r"Used (\d+) registers.*?(\d+) bytes smem", line)
        if m and name:
            res.setdefault(name, {}).update({"registers": int(m.group(1)), "static_smem_bytes": int(m.group(2))})
    return res


def step_times(rounds, steps, dev):
    import torch
    from moco_b200 import encoders
    from moco_b200.augment import augment_two_crop
    from moco_b200.NCE import MemoryMoCo
    from moco_b200.train_step import MoCoStep
    from moco_b200.util import moment_update
    batches = [batch("V2", 10 + b)[0] for b in range(4)]
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True

    def make(mlp):
        torch.manual_seed(0)
        model = encoders.resnet50(low_dim=128, mlp=mlp).to(dev).to(memory_format=torch.channels_last)
        ema = encoders.resnet50(low_dim=128, mlp=mlp).to(dev).to(memory_format=torch.channels_last)
        moment_update(model, ema, 0)
        contrast = MemoryMoCo(128, K, 0.2).to(dev)
        opt = torch.optim.SGD(model.parameters(), lr=BATCH / 256 * 0.03, momentum=0.9, weight_decay=1e-4)
        return MoCoStep(model, ema, contrast, opt, channels_last=True)

    arms = {"fc": make(False), "mlp": make(True)}
    sums = torch.zeros(2, device=dev)

    def run(step, n):
        for b in itertools.islice(itertools.cycle(batches), n):
            x1, x2 = torch.split(augment_two_crop(b), [3, 3], dim=1)
            loss, prob = step(x1, x2, 1)
            sums[0].add_(loss.detach(), alpha=BATCH)
            sums[1].add_(prob.detach(), alpha=BATCH)

    for step in arms.values():
        run(step, 3)
    times, clocks = {name: [] for name in arms}, []
    for _ in range(rounds):
        for name, step in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(step, steps)
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) / steps * 1e3)
            clocks.append(sm_clock())
    res = {name: {"ms_per_step": [round(t, 3) for t in ts], "median_ms": round(statistics.median(ts), 3)}
           for name, ts in times.items()}
    res.update({"mlp_minus_fc_ms": round(res["mlp"]["median_ms"] - res["fc"]["median_ms"], 3), "rounds": rounds,
                "steps_per_round": steps, "sm_mhz_after_each_window": clocks, "arch": "resnet50", "batch": BATCH,
                "nce_k": K, "aug": "V2"})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "moco_augment_v2_times"))
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("augment_v2_times: needs a CUDA device")
    dev = torch.device("cuda", 0)
    res = {"card": card(), "augment": augment_times(args.rounds, args.iters, dev), "ptxas": ptxas()}
    res["recipe_step"] = step_times(args.rounds, args.steps, dev)
    res["card_after"] = card()
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "augment_v2_times_h100.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
