"""Time moco_conv1x1_dgrad_bn_bwd + moco_bn_bwd_apply_given against cuDNN's 1x1 dgrad + moco_bn_add_relu_bwd2 on
every shape of ResNet-50 that bn._dgrad_bn_bwd can take at batch 256: the input gradient of a conv1 whose input is
an identity block's output, and that block's residual BatchNorm backward.

CUDA events around `--iters` calls of each path, the two paths alternated, best of `--rounds`.  Algorithmic bytes:
    fused:   dH, w read; x, dy2, mask read, g written (dgrad kernel); g, x read, dx written (apply)
    unfused: dH, w read, dX written (dgrad); bwd2 reads dX, dy2, x, mask twice, writes dx and dres
Prints one JSON line and writes it to --out.

    python tools/conv1x1_dgrad_times.py [--batch 256] [--iters 50] [--rounds 2] [--out FILE]
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

# (C, Cout, H): the block output's channels (= conv1's Cin), conv1's Cout, and the spatial size at 224^2 input
SHAPES = [(256, 64, 56), (256, 128, 56), (512, 128, 28), (512, 256, 28)]
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
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from moco_b200 import _lib
    from moco_b200.bn import _layer
    if not torch.cuda.is_available():
        raise SystemExit("conv1x1_dgrad_times.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.backends.cudnn.benchmark = False               # bench.py's settings
    torch.backends.cudnn.deterministic = True
    lib = _lib.load()
    cl = torch.channels_last
    ws_bn = torch.zeros(lib.moco_bn_workspace_bytes(), dtype=torch.uint8, device=dev)
    ws_cv = torch.zeros(lib.moco_conv1x1_workspace_bytes(), dtype=torch.uint8, device=dev)
    rows = []
    for C, Cout, H in SHAPES:
        N = args.batch
        M = N * H * H
        g = torch.Generator(device=dev).manual_seed(C + Cout)
        t = lambda c: torch.randn((N, c, H, H), device=dev, generator=g).bfloat16().contiguous(memory_format=cl)
        dh, x, dy2 = t(Cout), t(C), t(C)
        w = (torch.randn((Cout, C, 1, 1), device=dev, generator=g) * Cout ** -0.5).bfloat16()
        mask = torch.randint(0, 256, (M, C // 8), dtype=torch.uint8, device=dev, generator=g)
        gamma = torch.rand(C, device=dev, generator=g) + 0.5
        mean, invstd = torch.randn(C, device=dev, generator=g), torch.rand(C, device=dev, generator=g) + 0.5
        f32 = lambda: torch.empty(C, dtype=torch.float32, device=dev)
        dg, db = f32(), f32()
        bn = _layer(gamma, None, mean, invstd, dgamma=dg, dbeta=db)
        gbuf, dx, dres = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
        s = _lib.cur_stream()

        def fused():
            _lib.check(lib.moco_conv1x1_dgrad_bn_bwd(dh.data_ptr(), w.data_ptr(), gbuf.data_ptr(), M, C, Cout,
                                                     x.data_ptr(), mask.data_ptr(), dy2.data_ptr(), None, bn, None,
                                                     ws_cv.data_ptr(), ws_cv.numel(), s), "dgrad_bn_bwd")
            _lib.check(lib.moco_bn_bwd_apply_given(gbuf.data_ptr(), x.data_ptr(), None, M, C, bn, None, dx.data_ptr(),
                                                   None, s), "apply_given")

        def unfused():
            dX = torch.ops.aten.convolution_backward(dh, x, w, None, [1, 1], [0, 0], [1, 1], False, [0, 0], 1,
                                                     [True, False, False])[0]
            _lib.check(lib.moco_bn_add_relu_bwd2(dX.data_ptr(), dy2.data_ptr(), x.data_ptr(), None, mask.data_ptr(), M,
                                                 C, bn, None, dx.data_ptr(), dres.data_ptr(), ws_bn.data_ptr(),
                                                 ws_bn.numel(), s), "bwd2")

        def timed(fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) * 1e3 / args.iters

        for _ in range(5):
            fused()
            unfused()
        torch.cuda.synchronize()
        best_f, best_u = float("inf"), float("inf")
        for _ in range(args.rounds):
            best_u = min(best_u, timed(unfused))
            best_f = min(best_f, timed(fused))
        E = M * C
        b_fused = 2 * M * Cout + 2 * C * Cout + E * (2 + 2 + 0.125 + 2) + E * (2 + 2 + 2)
        b_unfused = 2 * M * Cout + 2 * C * Cout + 2 * E + 2 * E * (2 + 2 + 2 + 0.125) + 2 * 2 * E
        rows.append({"C": C, "Cout": Cout, "M": M, "fused_us": round(best_f, 1), "unfused_us": round(best_u, 1),
                     "speedup": round(best_u / best_f, 3),
                     "fused_bytes": int(b_fused), "unfused_bytes": int(b_unfused),
                     "fused_GBps": round(b_fused / best_f * 1e-3, 1), "unfused_GBps": round(b_unfused / best_u * 1e-3, 1),
                     "fused_frac_hbm": round(b_fused / (best_f * 1e-6) / HBM, 3),
                     "unfused_frac_hbm": round(b_unfused / (best_u * 1e-6) / HBM, 3)})
        del dh, x, dy2, gbuf, dx, dres, mask
        torch.cuda.empty_cache()
    name, watts = card()
    line = {"what": "moco_conv1x1_dgrad_bn_bwd + moco_bn_bwd_apply_given vs cuDNN 1x1 dgrad + moco_bn_add_relu_bwd2, "
                    f"batch {args.batch}, best of {args.rounds} x {args.iters} calls (CUDA events, alternated)",
            "gpu": name or torch.cuda.get_device_name(dev), "power_limit_w": watts, "shapes": rows}
    print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(line, indent=1) + "\n")


if __name__ == "__main__":
    main()
