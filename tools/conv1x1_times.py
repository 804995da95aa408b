"""Time moco_conv1x1_bn_stats + the BatchNorm apply pass against cuDNN's 1x1 convolution + moco_bn_fwd_train
(statistics + apply) at every stride-1 1x1 convolution shape of ResNet-50's bottleneck blocks, and print one JSON line.

Each arm runs the convolution and the following training BatchNorm (ReLU, no residual) on the same seeded bf16
channels_last input, timed with CUDA events over `--iters` back-to-back calls after `--warmup` calls.  Rates are
algorithmic: FLOP = 2 M Cin Cout; bytes = x + w + y (+ y read by the statistics pass, old arm) + the apply pass
(y read, output written).  Peaks are the H100 SXM data sheet's (989 TFLOP/s dense bf16, 3.35 TB/s).

    python tools/conv1x1_times.py [--batch 256] [--iters 50] [--warmup 10] [--out FILE]
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

# (spatial side at batch 256, Cin, Cout, count per encoder, stride) of ResNet-50's 1x1 convolutions
SHAPES = [
    (56, 64, 64, 1, 1), (56, 256, 64, 2, 1), (56, 64, 256, 4, 1),
    (56, 256, 128, 1, 1), (28, 512, 128, 3, 1), (28, 128, 512, 4, 1), (28, 256, 512, 1, 2),
    (28, 512, 256, 1, 1), (14, 1024, 256, 5, 1), (14, 256, 1024, 6, 1), (14, 512, 1024, 1, 2),
    (14, 1024, 512, 1, 1), (7, 2048, 512, 2, 1), (7, 512, 2048, 3, 1), (7, 1024, 2048, 1, 2),
]
PEAK_TFLOPS, PEAK_GBS = 989.0, 3350.0


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
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import torch.nn.functional as F
    from moco_b200 import _lib
    from moco_b200 import bn as bn_mod

    if not torch.cuda.is_available():
        raise SystemExit("conv1x1_times.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    lib = _lib.load()
    cl = torch.channels_last
    gen = torch.Generator(device=dev).manual_seed(0)
    rows = []
    for side, cin, cout, count, stride in SHAPES:
        N = args.batch
        H = side * stride
        x = torch.randn(N, cin, H, H, device=dev, generator=gen).to(torch.bfloat16).contiguous(memory_format=cl)
        w = (torch.randn(cout, cin, 1, 1, device=dev, generator=gen) * cin ** -0.5).to(torch.bfloat16)
        M = N * side * side
        row = {"M": M, "Cin": cin, "Cout": cout, "count": count, "stride": stride}
        if stride != 1:
            row["new"] = "not handled (stride 2)"
            rows.append(row)
            continue
        bnm = bn_mod.BatchNormAct2d(cout, relu=True).to(dev)
        gamma, beta = bnm.weight.detach(), bnm.bias.detach()
        rm, rv, nbt = bnm.running_mean, bnm.running_var, bnm.num_batches_tracked
        stats = (rm, rv, nbt, 0.1, 1e-5)
        y = torch.empty((N, cout, side, side), dtype=torch.bfloat16, device=dev, memory_format=cl)
        out = torch.empty_like(y)
        mean = torch.empty(cout, dtype=torch.float32, device=dev)
        invstd = torch.empty_like(mean)
        ws_bn = bn_mod._workspace(dev)
        ws_cv = bn_mod._workspace(dev, conv=True)
        layer = bn_mod._layer(gamma, beta, mean, invstd, stats)
        stream = _lib.cur_stream()

        def new():
            _lib.check(lib.moco_conv1x1_bn_stats(x.data_ptr(), w.data_ptr(), y.data_ptr(), M, cin, cout, layer,
                                                 ws_cv.data_ptr(), ws_cv.numel(), stream), "conv1x1")
            _lib.check(lib.moco_bn_fwd_train_given(y.data_ptr(), None, out.data_ptr(), None, M, cout, 1, layer, None,
                                                   _lib.BN_STATS_GIVEN, None, 0, stream), "apply")

        def old():
            yy = F.conv2d(x, w)
            _lib.check(lib.moco_bn_fwd_train(yy.data_ptr(), None, out.data_ptr(), M, cout, gamma.data_ptr(),
                                             beta.data_ptr(), rm.data_ptr(), rv.data_ptr(), nbt.data_ptr(), 0.1, 1e-5,
                                             1, mean.data_ptr(), invstd.data_ptr(), ws_bn.data_ptr(), ws_bn.numel(),
                                             stream), "bn")

        def conv_only():
            F.conv2d(x, w)

        def timed(fn):
            for _ in range(args.warmup):
                fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) * 1e3 / args.iters

        flop = 2.0 * M * cin * cout
        io = 2.0 * (M * cin + cin * cout + M * cout)           # the GEMM's x, w, y
        apply_b = 2.0 * 2 * M * cout                            # apply: read y, write the output
        # alternate the arms twice; keep each arm's best
        t_new = t_old = t_conv = float("inf")
        for _ in range(2):
            t_new = min(t_new, timed(new))
            t_old = min(t_old, timed(old))
            t_conv = min(t_conv, timed(conv_only))
        row.update({
            "new_us": t_new, "old_us": t_old, "cudnn_conv_us": t_conv, "speedup": t_old / t_new,
            "new_tflops": flop / t_new / 1e6, "new_GB_s": (io + apply_b) / t_new / 1e3,
            "old_GB_s": (io + 2.0 * M * cout + apply_b) / t_old / 1e3,
            "new_frac_of_peak": max(flop / PEAK_TFLOPS / 1e6, (io + apply_b) / PEAK_GBS / 1e3) / t_new,
            "bound": "flop" if flop / PEAK_TFLOPS / 1e6 > (io + apply_b) / PEAK_GBS / 1e3 else "hbm",
        })
        rows.append(row)
        print(json.dumps(row), file=sys.stderr)
        del x, y, out
    gpu, watts = card()
    line = {"what": "moco_conv1x1_bn_stats + apply vs cuDNN 1x1 conv + moco_bn_fwd_train (statistics + apply), "
                    f"batch {args.batch}, CUDA events over {args.iters} calls, best of 2 alternations",
            "gpu": gpu or torch.cuda.get_device_name(dev), "power_limit_w": watts,
            "peaks": {"tflops_bf16_dense": PEAK_TFLOPS, "hbm_GB_s": PEAK_GBS, "source": "H100 SXM data sheet"},
            "shapes": rows}
    s = json.dumps(line)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
