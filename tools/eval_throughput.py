"""Throughput of the linear-evaluation step (eval.py:254-311) on one GPU, three arms alternated in one process.

Each step: the reference's fp32 NCHW [256, 3, 224, 224] batch -> frozen ResNet-50 forward to layer 6 (no grad) ->
LinearClassifierResNet(6, 1000) -> cross-entropy -> classifier backward + SGD (lr 30, momentum 0.9).  Arms:
  a  today's eval path: the unfrozen model in eval mode, bf16 autocast, channels_last, fed the same space-to-depth
     input pass as b, so that only the BatchNorm side differs (nn.BatchNorm2d, separate add and ReLU, materialised
     shortcut BN and stem BN outputs, torch average pool);
  b  the frozen path: MoCoResNet.freeze() and model(x, 6) (eval kernels, shortcut BN and average pool folded in);
  c  for context, the fp32 NCHW sequence the reference runs at --amp-opt-level O0.
The encoders run on fixed, deterministic cuDNN algorithms (as bench.py does).  After the timed rounds, a separate
torch.profiler pass (CUDA activities) gives each arm's device time per step by kernel class.  Prints one JSON line:
the card and its power limit, img/s per arm and round, the algorithmic BatchNorm-side bytes per step of each arm
(computed from the shapes below), the largest |difference| between the layer-6 features of a and b, and the time
and achieved bandwidth of arm b's pooled last-block kernel, the one a small per-GPU batch starves first.

    python tools/eval_throughput.py [--rounds 3] [--steps 20] [--warmup 5] [--batch 256]
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def bn_bytes(model, N, H, W, esize, fused):
    """Algorithmic bytes per forward moved around the BatchNorms (x / residual reads, y writes, the stem pool's read
    and write, the average pool's read and write) of a MoCoResNet at [N, 3, H, W]."""
    from moco_b200 import encoders
    total = 0
    H, W = (H - 1) // 2 + 1, (W - 1) // 2 + 1                  # stem conv, stride 2
    stem = N * H * W * 64
    H, W = (H - 1) // 2 + 1, (W - 1) // 2 + 1                  # max pool
    if fused:
        total += stem * esize + N * H * W * 64 * esize        # one pass: read x, write the pooled y
    else:
        total += stem * esize * 2 * 2 + stem * esize + N * H * W * 64 * esize   # BN, ReLU, pool
    blocks = list(model.layers)
    for i, b in enumerate(blocks):
        bottleneck = isinstance(b, encoders._Bottleneck)
        s = (b.conv2 if bottleneck else b.conv1).stride[0]
        Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
        inner = [N * H * W * b.bn1.num_features] if bottleneck else []
        inner.append(N * Ho * Wo * b.bn2.num_features if bottleneck else N * Ho * Wo * b.bn1.num_features)
        last = (b.bn3 if bottleneck else b.bn2).num_features
        m = N * Ho * Wo * last
        pooled = i == len(blocks) - 1
        if fused:
            total += sum(inner) * esize * 2                    # read x, write y
            total += m * esize * 2                             # read x, read the residual (or raw shortcut)
            total += N * last * 4 if pooled else m * esize     # fp32 features, or the map
        else:
            total += sum(inner) * esize * 4                    # BN read + write, ReLU read + write
            if b.short is not None:
                total += m * esize * 2                         # the shortcut BN's own pass
            total += m * esize * (2 + 3 + 2)                   # BN, add (two reads, one write), ReLU
            if pooled:
                total += m * esize + N * last * esize          # the average pool's read and write
        H, W = Ho, Wo
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--bytes-only", action="store_true", help="print the byte counts and exit (no GPU needed)")
    args = ap.parse_args()

    import torch
    from moco_b200 import encoders
    from moco_b200.linear_eval import LinearClassifierResNet
    N = args.batch
    proto = encoders.resnet50()
    nbytes = {"a": bn_bytes(proto, N, 224, 224, 2, False), "b": bn_bytes(proto, N, 224, 224, 2, True),
              "c": bn_bytes(proto, N, 224, 224, 4, False)}
    if args.bytes_only:
        print(json.dumps({"bn_side_bytes_per_step": nbytes}))
        return
    if not torch.cuda.is_available():
        raise SystemExit("eval_throughput.py needs a CUDA device")
    from step_profile import card, classify
    from torch.profiler import ProfilerActivity, profile
    from moco_b200.util import crop_to_s2d_bf16

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    gpu, watts = card()

    torch.manual_seed(0)
    cl = torch.channels_last
    m_a = encoders.resnet50().to(dev).to(memory_format=cl).eval()
    m_b = encoders.resnet50().to(dev).to(memory_format=cl)
    m_b.load_state_dict(m_a.state_dict())
    m_b.freeze()
    m_c = encoders.resnet50().to(dev).eval()
    m_c.load_state_dict(m_a.state_dict())
    for m in (m_a, m_c):
        m.requires_grad_(False)
    heads = {}
    for k in "abc":
        torch.manual_seed(1)
        h = LinearClassifierResNet(6, 1000).to(dev)
        heads[k] = (h, torch.optim.SGD(h.parameters(), lr=30.0, momentum=0.9, weight_decay=0.0))
    gen = torch.Generator(device=dev).manual_seed(1234)
    x = torch.randn(N, 3, 224, 224, device=dev, generator=gen)
    y = torch.randint(0, 1000, (N,), device=dev, generator=gen)
    crit = torch.nn.CrossEntropyLoss()

    def feats(arm):
        with torch.no_grad():
            if arm == "c":
                return m_c(x, 6)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                return (m_a(crop_to_s2d_bf16(x), 6) if arm == "a" else m_b(x, 6)).float()

    def step(arm):
        h, opt = heads[arm]
        loss = crit(h(feats(arm)), y)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()

    fa, fb = feats("a"), feats("b")
    max_abs = float((fa - fb).abs().max())
    rel = float((fa - fb).norm() / fa.norm())
    for arm in "abc":
        for _ in range(args.warmup):
            step(arm)
    torch.cuda.synchronize()
    runs = collections.defaultdict(list)
    for _ in range(args.rounds):
        for arm in "abc":
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step(arm)
            e1.record()
            torch.cuda.synchronize()
            runs[arm].append(N * args.steps * 1e3 / e0.elapsed_time(e1))

    split = {}
    for arm in "abc":
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.profile_steps):
                step(arm)
            torch.cuda.synchronize()
        us = collections.defaultdict(float)
        for ev in prof.events():
            if ev.device_time > 0:
                name = ev.name
                if "bn_eval_avgpool" in name:
                    cls = "bn_eval_avgpool"
                elif "bn_eval" in name or ("maxpool" in name and arm == "b"):
                    cls = "bn_eval"
                else:
                    cls = classify(name)
                us[cls] += ev.device_time
        split[arm] = {c: round(us[c] / 1e3 / args.profile_steps, 3) for c in sorted(us, key=lambda c: -us[c])}

    pool_ms = split["b"].get("bn_eval_avgpool", 0.0)
    last = m_b.layers[-1].bn3.num_features
    pool_bytes = N * 7 * 7 * last * 2 * 2 + N * last * 4
    print(json.dumps({
        "what": f"linear-eval step on 1 GPU: ResNet-50 frozen forward to layer 6 + linear classifier (2048 -> 1000) "
                f"+ CE + classifier backward + SGD, {N} img at 224x224; {args.rounds} alternated rounds of "
                f"{args.steps} steps per arm after {args.warmup} warm-up steps; deterministic cuDNN algorithms",
        "gpu": gpu or torch.cuda.get_device_name(dev), "power_limit_w": watts,
        "arms": {"a": "unfrozen eval model, bf16 autocast, channels_last (today's eval path)",
                 "b": "frozen model (eval kernels), bf16 autocast, channels_last",
                 "c": "fp32 NCHW, the reference's O0 sequence"},
        "img_per_s": dict(runs),
        "bn_side_bytes_per_step": nbytes,
        "features_a_vs_b": {"max_abs_diff": max_abs, "rel_l2_diff": rel},
        "kernel_ms_per_step_by_class": split,
        # the last block's BatchNorm + add + ReLU + average pool (arm b): reads x and the identity residual, writes
        # the fp32 features; its parallelism is N * C / 8 threads, so it is the kernel a small batch starves first
        "avgpool_kernel": {"us": round(pool_ms * 1e3, 2), "bytes": pool_bytes,
                           "GB_per_s": round(pool_bytes / (pool_ms * 1e-3) / 1e9, 1) if pool_ms else None},
    }))


if __name__ == "__main__":
    main()
