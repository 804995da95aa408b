"""Time moco_conv1x1_bn_add_relu_fwd against moco_conv1x1_bn_stats + moco_bn_fwd_train_given on every conv3 -> bn3 of
ResNet-50's bottlenecks that moco_conv1x1_bn_stats takes, at batch 256, in both modes bn.conv1x1_bn_add_relu uses:
    query: the statistics pass writes h = conv3(a2) (bn3's backward reads it); the apply writes y and the mask bits.
           today = stats(a2 -> h) + apply(h, r -> y, mask);  new = stats(a2 -> h) + recompute(a2, r -> y, mask)
    key:   no backward.  today = stats(a2 -> h) + apply(h, r -> y);  new = stats(a2, no store) + recompute(a2, r -> y)
Each shape runs with an identity residual and with a shortcut BN ("sc"); the shortcut's statistics pass runs inside
the apply call, as in stages 2-3 where the stride-2 shortcut convolution is cuDNN's.

CUDA events around `--iters` calls of each arm, the four arms alternated, best of `--rounds`.  Algorithmic bytes
(bf16, E = M * Cout elements, A = M * Cin):
    today: 2A + 2E (stats) + 6E (+ E/8 mask) (apply) (+ 2E shortcut statistics)
    new query: 2A + 2E (stats) + 2A + 4E (+ E/8) (recompute) (+ 2E);  new key: 2A + 2A + 4E (+ 2E)
Prints one JSON line and writes it to --out.

    python tools/conv1x1_apply_times.py [--batch 256] [--iters 50] [--rounds 3] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# (Cin, Cout, H): conv3's input channels (the bottleneck's width), output channels, spatial size at 224^2 input
SHAPES = [(64, 256, 56), (128, 512, 28), (256, 1024, 14)]
HBM = 3.35e12                                            # H100 SXM data sheet


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, watts = (s.strip() for s in out.split(","))
        return name, float(watts)
    except Exception:
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from moco_b200 import _lib
    from moco_b200.bn import _layer
    if not torch.cuda.is_available():
        raise SystemExit("conv1x1_apply_times.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    lib = _lib.load()
    cl = torch.channels_last
    ws = torch.zeros(max(lib.moco_bn_workspace_bytes(), lib.moco_conv1x1_workspace_bytes()), dtype=torch.uint8,
                     device=dev)
    ws_cv = torch.zeros(lib.moco_conv1x1_workspace_bytes(), dtype=torch.uint8, device=dev)
    GIVEN, SC_GIVEN = _lib.BN_STATS_GIVEN, _lib.BN_SC_STATS_GIVEN
    rows = []
    for Cin, C, H in SHAPES:
        for shortcut in (False, True):
            N = args.batch
            M = N * H * H
            g = torch.Generator(device=dev).manual_seed(Cin + C + shortcut)
            t = lambda c: torch.randn((N, c, H, H), device=dev, generator=g).bfloat16().contiguous(memory_format=cl)
            a2, r = t(Cin), t(C)
            w = (torch.randn((C, Cin, 1, 1), device=dev, generator=g) * Cin ** -0.5).bfloat16()
            h, y = torch.empty((N, C, H, H), dtype=torch.bfloat16, device=dev, memory_format=cl), t(C)
            mask = torch.empty((M, C // 8), dtype=torch.uint8, device=dev)
            f32 = lambda: torch.empty(C, dtype=torch.float32, device=dev)
            gamma, beta = torch.rand(C, device=dev, generator=g) + 0.5, torch.randn(C, device=dev, generator=g)
            rm, rv, nbt = torch.zeros(C, device=dev), torch.ones(C, device=dev), torch.zeros((), dtype=torch.long,
                                                                                              device=dev)
            stats = (rm, rv, nbt, 0.1, 1e-5)
            mean, invstd, mean2, invstd2 = f32(), f32(), f32(), f32()
            bn = _layer(gamma, beta, mean, invstd, stats)
            rm2, rv2 = rm.clone(), rv.clone()             # kept alive: the layer holds raw pointers
            sc = _layer(gamma, beta, mean2, invstd2, (rm2, rv2, None, 0.1, 1e-5)) if shortcut else None
            s = _lib.cur_stream()
            pw = ws.data_ptr(), ws.numel()

            def stats_pass():
                _lib.check(lib.moco_conv1x1_bn_stats(a2.data_ptr(), w.data_ptr(), h.data_ptr(), M, Cin, C, bn,
                                                     ws_cv.data_ptr(), ws_cv.numel(), s), "stats")

            def today(m):
                stats_pass()
                _lib.check(lib.moco_bn_fwd_train_given(h.data_ptr(), r.data_ptr(), y.data_ptr(), m, M, C, 1, bn, sc,
                                                       GIVEN, *pw, s), "fwd_given")

            def new_query():
                stats_pass()
                _lib.check(lib.moco_conv1x1_bn_add_relu_fwd(a2.data_ptr(), w.data_ptr(), r.data_ptr(), y.data_ptr(),
                                                            mask.data_ptr(), M, Cin, C, bn, sc, GIVEN, *pw, s), "new")

            def new_key():
                _lib.check(lib.moco_conv1x1_bn_add_relu_fwd(a2.data_ptr(), w.data_ptr(), r.data_ptr(), y.data_ptr(),
                                                            None, M, Cin, C, bn, sc, 0, *pw, s), "new")

            arms = {"today_query": lambda: today(mask.data_ptr()), "new_query": new_query,
                    "today_key": lambda: today(None), "new_key": new_key}

            def timed(fn):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                return e0.elapsed_time(e1) * 1e3 / args.iters

            for _ in range(5):
                for fn in arms.values():
                    fn()
            torch.cuda.synchronize()
            best = {k: float("inf") for k in arms}
            for _ in range(args.rounds):
                for k, fn in arms.items():
                    best[k] = min(best[k], timed(fn))
            A, E = 2 * M * Cin, 2 * M * C
            scb = E if shortcut else 0
            nbytes = {"today_query": A + E + 3 * E + E / 16 + scb, "new_query": A + E + A + 2 * E + E / 16 + scb,
                      "today_key": A + E + 3 * E + scb, "new_key": 2 * A + 2 * E + scb}
            row = {"Cin": Cin, "Cout": C, "M": M, "shortcut": shortcut}
            for k in arms:
                row[k + "_us"] = round(best[k], 1)
                row[k + "_GBps"] = round(nbytes[k] / best[k] * 1e-3, 1)
                row[k + "_frac_hbm"] = round(nbytes[k] / (best[k] * 1e-6) / HBM, 3)
            row["speedup_query"] = round(best["today_query"] / best["new_query"], 3)
            row["speedup_key"] = round(best["today_key"] / best["new_key"], 3)
            rows.append(row)
            del a2, r, h, y, mask
            torch.cuda.empty_cache()
    name, watts = card()
    line = {"what": "moco_conv1x1_bn_add_relu_fwd vs moco_conv1x1_bn_stats + moco_bn_fwd_train_given (conv3 -> bn3), "
                    f"batch {args.batch}, best of {args.rounds} x {args.iters} calls (CUDA events, arms alternated)",
            "gpu": name or torch.cuda.get_device_name(dev), "power_limit_w": watts, "shapes": rows}
    print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(line, indent=1) + "\n")


if __name__ == "__main__":
    main()
