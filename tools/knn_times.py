"""Cost of the weighted kNN evaluation on the GPU.

  - moco_knn (moco_b200.knn.knn_predict) at ImageNet's train-set size, Nb = 1,281,167 bank rows, Nq = 256 queries,
    k = 200, T = 0.07, for C = 128 (layer 7) and C = 2048 (layer 6), alternated with reference_knn (torch: fp32 mm,
    a stable sort in the contract's order, the vote) on the same inputs.  CUDA events around each call, `--iters`
    calls per arm after one warm-up call of each.  The features lie on a grid where every dot product is exact in
    fp32 ({-2, ..., 2} times a power of two that makes the rows about unit norm, as L2-normalised features are, so no
    vote weight falls into fp32's subnormal range), so both arms must give the same neighbours and predictions; that
    is checked.  Algorithmic rates: 2 Nq Nb C
    FLOP per sweep, two sweeps, and the bank's Nb C 2 bytes read per sweep.
  - The wall time of one examples/eval_knn.py run over a seeded synthetic JPEG folder written under the output
    directory (`--images` train images, a quarter as many val images, 10 classes, a randomly initialised checkpoint).
Writes one JSON object with the card's name, power limit and SM clock read in the same run.

    python tools/knn_times.py --out DIR [--iters 10] [--images 2048]
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
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, watts, sm, sm_max = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit_w": float(watts), "sm_clock_mhz": float(sm), "sm_clock_max_mhz": float(sm_max)}
    except Exception:
        return {}


def timed(fn, iters):
    import torch
    ms = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return ms


def kernel_times(iters):
    import torch
    from moco_b200.knn import knn_predict, reference_knn
    nb, nq, k, t, n_classes = 1_281_167, 256, 200, 0.07, 1000
    rows = []
    for c in (128, 2048):
        g = torch.Generator(device="cuda").manual_seed(c)
        step = 2.0 ** -((c * 2).bit_length() // 2)                # {-2..2} * step: rows of about unit norm
        bank = (torch.randint(-2, 3, (nb, c), generator=g, device="cuda") * step).bfloat16()
        q = (torch.randint(-2, 3, (nq, c), generator=g, device="cuda") * step).bfloat16()
        labels = torch.randint(0, n_classes, (nb,), generator=g, device="cuda", dtype=torch.int32)
        mine = lambda: knn_predict(bank, labels, q, k, t, n_classes, return_neighbors=True)
        ref = lambda: reference_knn(bank, labels, q, k, t, n_classes)
        a, b = mine(), ref()                                       # warm-up, and the outputs compared
        same = {"indices": bool(torch.equal(a.indices, b.indices)), "sims": bool(torch.equal(a.sims, b.sims)),
                "pred": bool(torch.equal(a.pred, b.pred)),
                "scores_max_rel_diff": float(((a.scores - b.scores).abs() / b.scores.abs().clamp_min(1e-30)).max())}
        del a, b
        ms_mine, ms_ref = [], []
        for _ in range(iters):                                     # alternated
            ms_mine += timed(mine, 1)
            ms_ref += timed(ref, 1)
        med = lambda v: sorted(v)[len(v) // 2]
        flop = 2 * 2 * nq * nb * c
        bytes_ = 2 * nb * c * 2
        rows.append({"C": c, "Nb": nb, "Nq": nq, "k": k, "T": t, "moco_knn_ms": ms_mine, "reference_knn_ms": ms_ref,
                     "moco_knn_ms_median": med(ms_mine), "reference_knn_ms_median": med(ms_ref),
                     "moco_knn_tflops": flop / med(ms_mine) / 1e9, "moco_knn_bank_gb_per_s": bytes_ / med(ms_mine) / 1e6,
                     "speedup_median": med(ms_ref) / med(ms_mine), "outputs_equal": same, "clock_after": card()})
        del bank, q, labels
        torch.cuda.empty_cache()
    return rows


def jpeg_folder(root, n_train, n_val):
    import torch
    import torchvision
    g = torch.Generator().manual_seed(0)
    for split, n in (("train", n_train), ("val", n_val)):
        for c in range(10):
            os.makedirs(os.path.join(root, split, f"c{c}"), exist_ok=True)
        for i in range(n):
            h, w = (int(v) for v in torch.randint(200, 500, (2,), generator=g))
            img = torch.randint(0, 256, (3, h, w), generator=g, dtype=torch.uint8)
            data = torchvision.io.encode_jpeg(img, quality=90)
            with open(os.path.join(root, split, f"c{i % 10}", f"{i}.jpg"), "wb") as f:
                f.write(data.numpy().tobytes())


def program_time(out, n_images):
    import importlib.util
    import torch
    from moco_b200.encoders import resnet50
    root = os.path.join(out, "jpegs")
    jpeg_folder(root, n_images, n_images // 4)
    torch.manual_seed(0)
    ckpt = os.path.join(out, "random.pth")
    torch.save({"model": resnet50().state_dict(), "epoch": 0}, ckpt)
    spec = importlib.util.spec_from_file_location("eval_knn", os.path.join(ROOT, "examples", "eval_knn.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    workers = min(os.cpu_count() or 1, 16)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = mod.main(["--data-dir", root, "--pretrained-model", ckpt, "--num-workers", str(workers)])
    torch.cuda.synchronize()
    return {"train_images": n_images, "val_images": n_images // 4, "num_workers": workers,
            "wall_s": time.perf_counter() - t0, "result": res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--images", type=int, default=2048)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("knn_times: no CUDA device")
    out = args.out or tempfile.mkdtemp(prefix="knn_times_")
    os.makedirs(out, exist_ok=True)
    res = {"card": card(), "cpu_count": os.cpu_count(), "kernel": kernel_times(args.iters)}
    res["program"] = program_time(out, args.images)
    res["card_after"] = card()
    path = os.path.join(out, "knn_times.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
