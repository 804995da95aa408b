"""Device time of one benchmark step, grouped by kernel class: where the 1-GPU step of bench.py spends its time.

Runs bench.py's exact single-GPU step (same encoders, MoCoStep, head, optimizer, seeded inputs and fixed cuDNN
algorithms) for a few warm steps, then profiles `--steps` more under torch.profiler (CUDA activities only) in a run
of its own, and prints one JSON line: milliseconds and launches per step for each kernel class.

    python tools/step_profile.py [--steps 3] [--warmup 5] [--arch resnet50] [--batch 256]
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# (class, substrings of the kernel name); the first class with a matching substring wins
CLASSES = [
    # conv3 recomputed with bn3's apply in its epilogue; first, since its name contains "bn_apply_kernel"
    ("conv1x1_bn_apply", ("conv1x1_bn_apply_kernel",)),
    ("conv1x1_stats", ("conv1x1_stats_kernel",)),     # csrc/conv1x1_sm90.cu: 1x1 forward + the next BN's statistics
    # 1x1 dgrad + the producing BN's backward sums; before conv_dgrad, which takes any name containing "dgrad"
    ("conv1x1_dgrad_bn", ("conv1x1_dgrad_bn_bwd_kernel",)),
    ("bn_stats", ("bn_stats_kernel",)),
    ("bn_apply", ("bn_apply_kernel",)),
    ("bn_bwd_reduce", ("bn_bwd_reduce_kernel",)),
    ("bn_bwd_apply", ("bn_bwd_apply_kernel",)),
    ("maxpool", ("maxpool",)),
    ("head", ("nce_", "queue_enqueue", "shard_")),
    ("input_path", ("crop", "shuffle", "gather_rows", "s2d")),
    ("optimizer_ema", ("multi_tensor_apply", "sgd", "ema_", "foreach")),
    ("conv_dgrad", ("dgrad",)),
    ("conv_wgrad", ("wgrad",)),
    ("conv_fwd", ("fprop", "implicit_convolve", "conv2d", "convolve")),
    ("conv_other", ("cudnn", "xmma", "nchwToNhwc", "nhwcToNchw", "cutlass")),
    # cuDNN runs the 1x1 convolutions (forward, dgrad and wgrad alike) as nvjet GEMMs; the fc layer adds three small ones
    ("conv_1x1_nvjet", ("nvjet",)),
    ("gemm", ("gemm", "cublas")),
    ("aten_elementwise", ("elementwise", "vectorized", "unrolled")),
    ("aten_other", ("at::native",)),
    ("copies", ("Memcpy", "Memset")),
]


def classify(name: str) -> str:
    for cls, keys in CLASSES:
        if any(k in name for k in keys):
            return cls
    return "other"


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, watts = (s.strip() for s in out.split(","))
        return name, float(watts)
    except Exception:                                   # no nvidia-smi: the card name still comes from torch
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--arch", default="resnet50")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--feat-dim", type=int, default=128)
    ap.add_argument("--nce-k", type=int, default=16384)
    ap.add_argument("--nce-t", type=float, default=0.07)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from moco_b200 import encoders
    from moco_b200.NCE import MemoryMoCo
    from moco_b200.train_step import MoCoStep

    if not torch.cuda.is_available():
        raise SystemExit("step_profile.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    # bench.py's settings (run_native): fixed deterministic cuDNN algorithms, TF32 allowed
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True

    N, C, K, T = args.batch, args.feat_dim, args.nce_k, args.nce_t
    torch.manual_seed(0)
    ctor = getattr(encoders, args.arch)
    cl = torch.channels_last
    model = ctor(low_dim=C).to(dev).to(memory_format=cl)
    model_ema = ctor(low_dim=C).to(dev).to(memory_format=cl)
    model_ema.load_state_dict(model.state_dict())
    contrast = MemoryMoCo(C, K, T).to(dev)
    opt = torch.optim.SGD(model.parameters(), lr=0.03 * N / 256, momentum=0.9, weight_decay=1e-4)
    step = MoCoStep(model, model_ema, contrast, opt, channels_last=True)
    gen = torch.Generator(device=dev).manual_seed(1234)
    inputs = torch.randn(N, 6, 224, 224, device=dev, generator=gen)
    x1, x2 = torch.split(inputs, [3, 3], dim=1)

    for _ in range(args.warmup):
        step(x1, x2, 1)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step(x1, x2, 1)
    e1.record()
    torch.cuda.synchronize()
    ms_step = e0.elapsed_time(e1) / args.steps

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step(x1, x2, 1)
        torch.cuda.synchronize()
    us = collections.defaultdict(float)
    launches = collections.defaultdict(int)
    names = collections.defaultdict(lambda: collections.defaultdict(float))
    name_launches = collections.defaultdict(lambda: collections.defaultdict(int))
    pools = []                                          # (start, name, device us) of every max-pool launch
    for ev in prof.events():
        t = ev.device_time
        if t <= 0:
            continue
        cls = classify(ev.name)
        us[cls] += t
        launches[cls] += 1
        names[cls][ev.name] += t
        name_launches[cls][ev.name] += 1
        if cls == "maxpool":
            pools.append((ev.time_range.start, ev.name, t))
    # the stem's pool launches in step order (forward of each encoder, then the backward), with algorithmic GB/s:
    # input [N, H/2, W/2, 64] bf16 after the stride-2 stem convolution, pooled to [N, H/4, W/4, 64] + 1 tap byte each
    pools.sort()
    per_step = len(pools) // args.steps if args.steps else 0
    H = inputs.shape[-1] // 2
    Ho = (H - 1) // 2 + 1
    x_bytes, y_bytes = N * H * H * 64 * 2, N * Ho * Ho * 64 * 2
    maxpool_launches = []
    for i in range(per_step):
        runs = pools[i::per_step]
        name = runs[0][1]
        mean_us = sum(r[2] for r in runs) / len(runs)
        # forward: x, y + taps; backward: dy + taps (+ dy2, the kSum instance), dx
        nbytes = (x_bytes + y_bytes * 3 // 2) if "fwd" in name else (y_bytes * 3 // 2 + x_bytes)
        if "bwd_kernel<true>" in name:
            nbytes += y_bytes
        maxpool_launches.append({"kernel": name[:80], "us": mean_us, "bytes": nbytes, "GB_s": nbytes / mean_us / 1e3})
    total = sum(us.values())
    gpu, watts = card()
    line = {
        "what": f"device time per step by kernel class: bench.py's 1-GPU step ({args.arch}, {N} img, bf16, K={K}), "
                f"torch.profiler CUDA kernel records over {args.steps} steps after {args.warmup} warm-up steps",
        "gpu": gpu or torch.cuda.get_device_name(dev), "power_limit_w": watts,
        "ms_per_step_unprofiled": ms_step,
        "kernel_ms_per_step": total / 1e3 / args.steps,
        "classes": {c: {"ms_per_step": us[c] / 1e3 / args.steps, "launches_per_step": launches[c] / args.steps,
                        "share": us[c] / total}
                    for c in sorted(us, key=lambda c: -us[c])},
        # the kernels behind the catch-all classes, so that a misfiled kernel is visible
        "top_kernels": {c: [[n[:120], t / 1e3 / args.steps] for n, t in sorted(names[c].items(), key=lambda kv: -kv[1])[:4]]
                        for c in ("other", "aten_other", "conv_other", "gemm") if c in names},
        # every element-wise ATen kernel: [name, launches per step, ms per step]
        "aten_elementwise_kernels": [[n[:160], name_launches["aten_elementwise"][n] / args.steps, t / 1e3 / args.steps]
                                     for n, t in sorted(names["aten_elementwise"].items(), key=lambda kv: -kv[1])],
        "maxpool_launches": maxpool_launches,
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
