"""Device time and algorithmic bandwidth of the stem's max-pool kernels, next to bn_apply_kernel at the same size.

The stem of bench.py's ResNet-50 step runs three max-pool launches: the BatchNorm + ReLU + pool forward of each
encoder (moco_bn_relu_maxpool_fwd_train's second launch, tap bytes written by both) and the pool backward of the
query encoder.  This times every entry point that launches them at the stem's size ([N, 112, 112, 64] bf16 for
224-pixel images) on seeded inputs, warm, two ways:
  - CUDA events around `--iters` back-to-back calls of each entry point (per call);
  - torch.profiler kernel records over the same calls in a run of their own (per kernel, so that the pool launch
    of moco_bn_relu_maxpool_fwd_train is separated from its statistics pass).
Algorithmic bytes are what the kernel must move at least: every input read once, every output written once.  Prints
one JSON line with the card name, its power limit and the SM clock read in the same run.

    python tools/pool_times.py [--batch 256] [--hw 112] [--channels 64] [--iters 30]
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, watts, sm, sm_max = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit_w": float(watts), "sm_mhz": float(sm), "sm_max_mhz": float(sm_max)}
    except Exception:
        return {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--hw", type=int, default=112)
    ap.add_argument("--channels", type=int, default=64)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from moco_b200 import _lib
    from moco_b200.bn import _layer

    if not torch.cuda.is_available():
        raise SystemExit("pool_times.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lib = _lib.load()
    N, H, W, C = args.batch, args.hw, args.hw, args.channels
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    M, Mo = N * H * W, N * OH * OW
    g = torch.Generator(device=dev).manual_seed(7)
    cl = torch.channels_last
    bf = lambda *s: torch.randn(s, device=dev, generator=g).bfloat16().contiguous(memory_format=cl)
    x, dx = bf(N, C, H, W), bf(N, C, H, W)
    y, dy, dy2 = bf(N, C, OH, OW), bf(N, C, OH, OW), bf(N, C, OH, OW)
    taps = torch.empty((N, OH, OW, C), dtype=torch.uint8, device=dev)
    f32 = lambda: torch.ones(C, dtype=torch.float32, device=dev)
    w, b, mean, invstd = f32(), f32() * 0.0, f32(), f32()
    ws = torch.zeros(lib.moco_bn_workspace_bytes(), dtype=torch.uint8, device=dev)
    s = _lib.cur_stream()
    bn = _layer(w, b, mean, invstd, (None, None, None, 0.1, 1e-5))

    def ok(rc):
        if rc != 0:
            raise RuntimeError(lib.moco_last_error().decode())

    # (case, call, {kernel substring: algorithmic bytes of one launch})
    cases = [
        ("moco_bn_fwd_train", lambda: ok(lib.moco_bn_fwd_train(
            x.data_ptr(), None, dx.data_ptr(), M, C, w.data_ptr(), b.data_ptr(), None, None, None, 0.1, 1e-5, 1,
            mean.data_ptr(), invstd.data_ptr(), ws.data_ptr(), ws.numel(), s)),
         {"bn_apply_kernel": 2 * M * C * 2, "bn_stats_kernel": M * C * 2}),
        ("moco_bn_relu_maxpool_fwd_train", lambda: ok(lib.moco_bn_relu_maxpool_fwd_train(
            x.data_ptr(), y.data_ptr(), taps.data_ptr(), N, H, W, C, bn, ws.data_ptr(), ws.numel(), s)),
         {"maxpool3x3s2_fwd": M * C * 2 + Mo * C * 3, "bn_stats_kernel": M * C * 2}),
        ("moco_maxpool3x3s2_fwd", lambda: ok(lib.moco_maxpool3x3s2_fwd(
            x.data_ptr(), y.data_ptr(), taps.data_ptr(), N, H, W, C, s)),
         {"maxpool3x3s2_fwd": M * C * 2 + Mo * C * 3}),
        ("moco_maxpool3x3s2_bwd", lambda: ok(lib.moco_maxpool3x3s2_bwd(
            dy.data_ptr(), taps.data_ptr(), dx.data_ptr(), N, H, W, C, s)),
         {"maxpool3x3s2_bwd": Mo * C * 3 + M * C * 2}),
    ]
    if hasattr(lib, "moco_maxpool3x3s2_bwd2"):
        cases.append(("moco_maxpool3x3s2_bwd2", lambda: ok(lib.moco_maxpool3x3s2_bwd2(
            dy.data_ptr(), dy2.data_ptr(), taps.data_ptr(), dx.data_ptr(), N, H, W, C, s)),
            {"maxpool3x3s2_bwd": Mo * C * 5 + M * C * 2}))

    # the backward needs tap bytes of a real forward
    ok(lib.moco_maxpool3x3s2_fwd(x.data_ptr(), y.data_ptr(), taps.data_ptr(), N, H, W, C, s))
    result = {"what": f"stem max-pool kernels at [N={N}, {H}x{W}, C={C}] bf16 (OH x OW = {OH}x{OW}), "
                      f"{args.iters} warm calls each; GB/s = algorithmic bytes / kernel time",
              **card(), "calls": {}, "kernels": {}}
    for name, call, _ in cases:
        for _ in range(args.warmup):
            call()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            call()
        e1.record()
        torch.cuda.synchronize()
        result["calls"][name] = {"us_per_call_events": e0.elapsed_time(e1) * 1e3 / args.iters}

    for name, call, nbytes in cases:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                call()
            torch.cuda.synchronize()
        per = collections.defaultdict(list)
        for ev in prof.events():
            if ev.device_time > 0:
                per[ev.name].append(ev.device_time)
        for kname, times in per.items():
            key = next((k for k in nbytes if k in kname), None)
            if key is None:
                continue
            us = sum(times) / len(times)
            result["kernels"][f"{name}:{key}"] = {"us": us, "launches": len(times), "bytes": nbytes[key],
                                                  "GB_s": nbytes[key] / us / 1e3}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
