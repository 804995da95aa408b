"""Host side of the linear evaluation's real-data path, no GPU needed: the resize-window records equal torchvision's
Resize / CenterCrop arithmetic, ImageFolderEval's draws and records reproduce eval.py's train and validation Compose
bit for bit, the loader packs what decode_image returns, malformed records and bad C arguments are refused before
any launch, the learning-rate schedule equals the reference's, and the validation accounting over 2 and 3 gloo ranks
counts every sample exactly once and gives world 1's accuracy."""
import ctypes
import importlib.util
import os
import warnings

import numpy as np
import pytest
import torch
import torchvision
from torchvision import transforms as T
from torchvision.transforms import functional as TF

from moco_b200 import _lib
from moco_b200 import augment as A
from moco_b200 import linear_eval as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NORMALIZE = T.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])


def _image(h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8)


# --------------------------------------------------------------------------------------------------------------------
# records against torchvision

def _sizes():
    """About 200 (h, w): portrait, landscape and square; short side below, at and above 256; long sides of both
    parities after the resize (so both the exact and the half-to-even centre offsets occur)."""
    shorts = [64, 100, 143, 200, 224, 255, 256, 257, 300, 333, 375, 384, 480, 500, 512, 640, 768, 1000]
    ratios = [1.0, 1.001, 1.25, 4 / 3, 1.337, 1.5, 16 / 9, 2.0, 3.1, 5.0]
    out = set()
    for s in shorts:
        for r in ratios:
            long = int(s * r)
            out.add((s, long))
            out.add((long, s))
    out |= {(300, 400), (400, 300), (375, 500), (500, 375), (333, 500), (3000, 4000), (4000, 3000), (256, 256)}
    return sorted(out)


@pytest.mark.parametrize("resize,out", [(256, 224), (288, 256), (146, 128), (225, 224)])
def test_window_records_equal_torchvision_resize_and_center_crop(resize, out):
    sizes = _sizes()
    assert len(sizes) >= 190
    parities, half_to_even = set(), 0
    for h, w in sizes:
        rec = A.resize_window_params(h, w, resize, out).tolist()
        assert rec[:4] == [0, 0, h, w]
        rh, rw = T.Resize(resize)(torch.zeros(1, h, w, dtype=torch.uint8)).shape[1:]
        assert (rec[A.RESIZED_H], rec[A.RESIZED_W]) == (rh, rw), (h, w)
        coords = (torch.arange(rh, dtype=torch.int64).view(rh, 1) * rw + torch.arange(rw)).view(1, rh, rw)
        first = int(TF.center_crop(coords, [out, out])[0, 0, 0])
        assert (rec[A.WIN_TOP], rec[A.WIN_LEFT]) == divmod(first, rw), (h, w)
        parities.add(((rh - out) % 2, (rw - out) % 2))
        half_to_even += ((rh - out) % 2 == 1 and (rh - out) % 4 == 1) + ((rw - out) % 2 == 1 and (rw - out) % 4 == 1)
    assert {p[0] for p in parities} == {0, 1} and {p[1] for p in parities} == {0, 1}
    assert half_to_even > 0          # x.5 rounded down to the even integer


def test_half_to_even_offset_of_a_300_by_400_image():
    rec = A.resize_window_params(300, 400).tolist()
    assert rec[4:] == [256, 341, 16, 58]          # (341 - 224) / 2 = 58.5 -> 58, not 59
    rec = A.resize_window_params(400, 300).tolist()
    assert rec[4:] == [341, 256, 58, 16]
    assert A.resize_window_params(1000, 3).tolist()[4:6] == [int(256 * 1000 / 3), 256]


def test_window_that_does_not_fit_raises():
    with pytest.raises(ValueError, match="does not fit"):
        A.resize_window_params(300, 400, resize=200, out=224)
    with pytest.raises(ValueError):
        A.resize_window_params(0, 400)


# --------------------------------------------------------------------------------------------------------------------
# ImageFolderEval against eval.py's transforms (eval.py:92-116, as tensor ops)

def _eval_train_compose(aug, crop):
    if aug == "NULL":
        ts = [T.RandomResizedCrop(224, scale=(crop, 1.)), T.RandomHorizontalFlip()]
    else:
        ts = [T.RandomResizedCrop(224, scale=(crop, 1.)), T.RandomGrayscale(p=0.2), T.ColorJitter(0.4, 0.4, 0.4, 0.4),
              T.RandomHorizontalFlip()]
    return T.Compose(ts + [NORMALIZE])


def _eval_val_compose():
    return T.Compose([T.Resize(224 + 32), T.CenterCrop(224), NORMALIZE])


def _folder(root, split, sizes, classes=3, fmt="png", gray=()):
    for c in range(classes):
        os.makedirs(os.path.join(root, split, f"class{c}"), exist_ok=True)
    for i, (h, w) in enumerate(sizes):
        img = _image(h, w, seed=100 + i).permute(2, 0, 1).contiguous()
        if i in gray:
            img = img[:1].contiguous()
        data = torchvision.io.encode_png(img) if fmt == "png" else torchvision.io.encode_jpeg(img, quality=90)
        with open(os.path.join(root, split, f"class{i % classes}", f"img{i:03d}.{fmt}"), "wb") as f:
            f.write(data.numpy().tobytes())
    return os.path.join(root, split)


@pytest.mark.parametrize("aug", ["NULL", "CJ"])
def test_train_items_reproduce_eval_train_compose(tmp_path, aug):
    root = _folder(str(tmp_path), "train", [(97, 131), (300, 400), (40, 600)])
    ds = A.ImageFolderEval(root, train=True, scale=(0.2, 1.0), aug=aug)
    comp = _eval_train_compose(aug, 0.2)
    for k in range(len(ds)):
        path = ds.samples[k][0]
        x = torchvision.io.decode_image(path, mode=torchvision.io.ImageReadMode.RGB).float() / 255
        for seed in range(40):
            torch.manual_seed(seed)
            hwc, rec, target, index = ds[k]
            torch.manual_seed(seed)
            ref = comp(x)
            assert rec.shape == (1, A.WORDS) and index == k and target == ds.samples[k][1]
            assert torch.equal(A.reference_crop(hwc, rec[0]), ref), (aug, k, seed)


@pytest.mark.parametrize("aug", ["NULL", "CJ"])
def test_val_items_reproduce_eval_val_compose(tmp_path, aug):
    sizes = [(97, 131), (300, 400), (400, 300), (256, 256), (256, 301), (333, 500), (1100, 250)]
    root = _folder(str(tmp_path), "val", sizes)
    ds = A.ImageFolderEval(root, train=False, aug=aug)
    comp = _eval_val_compose()
    for k in range(len(ds)):
        hwc, rec, _, index = ds[k]
        assert rec.shape == (1, A.WIN_WORDS) and index == k
        x = hwc.permute(2, 0, 1).float() / 255
        assert torch.equal(A.reference_resize_center_crop(hwc, rec[0]), comp(x)), ds.samples[k][0]


def _old_two_crop_collate(items):
    """ImageFolderTwoCrop.collate_fn as it packed before the packing moved into pack_images."""
    sizes = [it[0].numel() for it in items]
    offsets = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    pixels = torch.cat([it[0].reshape(-1) for it in items])
    params = torch.cat([it[1] for it in items]).clone()
    off = np.repeat(offsets, 2)
    params[:, A.OFF_LO] = torch.from_numpy((off & 0xFFFFFFFF).astype(np.uint32).view(np.int32))
    params[:, A.OFF_HI] = torch.from_numpy((off >> 32).astype(np.int32))
    return pixels, params, torch.tensor([it[2] for it in items], dtype=torch.int64)


@pytest.mark.parametrize("fmt", ["png", "jpg"])
@pytest.mark.parametrize("train", [True, False])
def test_packing_targets_and_indices(tmp_path, fmt, train):
    sizes = [(64, 80), (97, 61), (260, 240), (33, 250), (300, 400), (90, 90)]
    root = _folder(str(tmp_path), "x", sizes, fmt=fmt, gray=(2,))
    ds = A.ImageFolderEval(root, train=train, aug="CJ")
    torch.manual_seed(3)
    order = [4, 0, 5, 2, 1, 3]
    items = [ds[i] for i in order]
    pixels, params, targets, indices = ds.collate_fn(items)
    words = A.WORDS if train else A.WIN_WORDS
    assert pixels.dtype == torch.uint8 and params.dtype == torch.int32 and params.shape == (len(order), words)
    assert indices.tolist() == order and targets.tolist() == [ds.samples[i][1] for i in order]
    off, gray_seen = 0, False
    for n, i in enumerate(order):
        dec = torchvision.io.decode_image(ds.samples[i][0], mode=torchvision.io.ImageReadMode.RGB).permute(1, 2, 0)
        h, w = dec.shape[:2]
        assert torch.equal(pixels[off:off + h * w * 3].view(h, w, 3), dec)
        r = params[n].tolist()
        assert r[A.OFF_LO] == off and r[A.OFF_HI] == 0 and (r[A.SRC_H], r[A.SRC_W]) == (h, w)
        if not train:
            assert r[4:] == A.resize_window_params(h, w).tolist()[4:]
        if ds.samples[i][0].endswith(f"img002.{fmt}"):                 # the grayscale file decodes to R = G = B
            px = pixels[off:off + h * w * 3].view(-1, 3)
            assert torch.equal(px[:, 0], px[:, 1]) and torch.equal(px[:, 0], px[:, 2])
            gray_seen = True
        off += h * w * 3
    assert off == pixels.numel() and gray_seen

    two = A.ImageFolderTwoCrop(root, aug="CJ")
    torch.manual_seed(4)
    items2 = [two[i] for i in order]
    got, want = A.ImageFolderTwoCrop.collate_fn(items2), _old_two_crop_collate(items2)
    assert all(torch.equal(a, b) for a, b in zip(got, want))


def test_eval_loader_batches_with_a_bound_collate(tmp_path):
    root = _folder(str(tmp_path), "val", [(50 + 7 * i, 300 - 3 * i) for i in range(5)])
    ds = A.ImageFolderEval(root, train=False)
    loader = torch.utils.data.DataLoader(ds, batch_size=2, num_workers=2, collate_fn=ds.collate_fn,
                                         sampler=L.ShardSampler(len(ds), 1, 2))
    seen = []
    for pixels, params, _, idx in loader:
        A.validate_windows(params, pixels.numel(), 224, 224, 256)
        seen += idx.tolist()
    assert seen == [1, 3]


# --------------------------------------------------------------------------------------------------------------------
# malformed records and the C entry's refusals

def _good_windows():
    a, b = A.resize_window_params(300, 400), A.resize_window_params(120, 100)
    pixels, params = A.pack_images([torch.zeros(300, 400, 3, dtype=torch.uint8),
                                    torch.zeros(120, 100, 3, dtype=torch.uint8)], [a[None], b[None]])
    return params, pixels.numel()


@pytest.mark.parametrize("word,value,match", [
    (A.OFF_LO, 300 * 400 * 3 + 1, "outside the pixel buffer"),
    (A.OFF_HI, -1, "outside the pixel buffer"),
    (A.SRC_H, 0, "image size"),
    (A.SRC_W, 101, "outside the pixel buffer"),
    (A.RESIZED_H, 0, "resized size"),
    (A.RESIZED_W, -3, "resized size"),
    (A.RESIZED_W, 200, "window outside"),
    (A.WIN_TOP, -1, "window outside"),
    (A.WIN_LEFT, 40, "window outside"),
    (A.WIN_TOP, 84, "window outside"),
])
def test_malformed_windows_raise_value_error(word, value, match):
    params, nbytes = _good_windows()
    A.validate_windows(params, nbytes, 224, 224, 256)
    bad = params.clone()
    bad[1, word] = value
    with pytest.raises(ValueError, match=match):
        A.validate_windows(bad, nbytes, 224, 224)


def test_window_downscale_limit_and_resize_check():
    params, _ = _good_windows()
    p = params[:1].clone()
    p[0, A.SRC_H], p[0, A.SRC_W] = 1, 1000 * 256
    p[0, A.RESIZED_H], p[0, A.RESIZED_W], p[0, A.WIN_TOP], p[0, A.WIN_LEFT] = 256, 256, 16, 16
    A.validate_windows(p, 10 ** 9, 224, 224, 256)
    p[0, A.SRC_W] = 1000 * 256 + 1
    with pytest.raises(ValueError, match="wider"):
        A.validate_windows(p, 10 ** 9, 224, 224)
    with pytest.raises(ValueError, match="short side"):
        A.validate_windows(params, 10 ** 7, 224, 224, resize=288)
    with pytest.raises(ValueError, match=r"int32 \[n, 8\]"):
        A.validate_windows(params[:, :7], 10 ** 7, 224, 224)


def test_resize_center_crops_refuses_a_cpu_device_and_bad_records():
    params, nbytes = _good_windows()
    with pytest.raises(RuntimeError, match="CUDA only"):
        A.resize_center_crops((torch.zeros(nbytes, dtype=torch.uint8), params), device="cpu")
    with pytest.raises(ValueError):
        A.resize_center_crops((torch.zeros(nbytes - 1, dtype=torch.uint8), params), device="cpu")


FAKE = 0x7f0000010000


def _args(**kw):
    norm = (ctypes.c_float * 6)(*A.MEAN, *A.STD)
    a = dict(pixels=FAKE, pixels_bytes=1000, windows=FAKE + 0x1000, n=2, out_h=224, out_w=224, norm=norm,
             dst=FAKE + 0x2000, dst_dtype=_lib.MOCO_BF16, stream=None)
    a.update(kw)
    return list(a.values())


@pytest.mark.parametrize("kw,match", [
    (dict(pixels=None), b"bad argument"),
    (dict(pixels_bytes=0), b"bad argument"),
    (dict(windows=None), b"bad argument"),
    (dict(windows=FAKE + 0x1004), b"bad argument"),
    (dict(dst=None), b"bad argument"),
    (dict(dst=FAKE + 0x2001), b"bad argument"),
    (dict(dst=FAKE + 0x2002, dst_dtype=_lib.MOCO_F32), b"bad argument"),
    (dict(dst_dtype=7), b"dst_dtype=7"),
    (dict(norm=None), b"bad argument"),
    (dict(norm=(ctypes.c_float * 6)(float("nan"), 0.4, 0.4, 0.2, 0.2, 0.2)), b"norm must be finite"),
    (dict(norm=(ctypes.c_float * 6)(0.4, 0.4, 0.4, 0.2, float("inf"), 0.2)), b"norm must be finite"),
    (dict(norm=(ctypes.c_float * 6)(0.4, 0.4, 0.4, 0.2, 0.0, 0.2)), b"std != 0"),
    (dict(out_h=0), b"out_h, out_w in [1, 1024]"),
    (dict(out_h=1025), b"out_h, out_w in [1, 1024]"),
    (dict(out_w=0), b"out_h, out_w in [1, 1024]"),
    (dict(out_w=1025), b"out_h, out_w in [1, 1024]"),
    (dict(n=-1), b"n in [0, 65535]"),
    (dict(n=65536), b"n in [0, 65535]"),
])
def test_resize_entry_refuses_bad_arguments_without_a_launch(kw, match):
    lib = _lib.load()
    before = _lib.launches
    assert lib.moco_resize_center_crops(*_args(**kw)) == -1, kw
    err = lib.moco_last_error()
    assert err.startswith(b"moco_resize_center_crops: ") and match in err, err
    assert _lib.launches == before


def test_resize_entry_with_no_images_launches_nothing():
    lib = _lib.load()
    before = _lib.launches
    assert lib.moco_resize_center_crops(*_args(n=0, pixels=None, windows=None, dst=None)) == 0
    assert _lib.launches == before


def test_header_record_layout_matches_the_host_words():
    text = open(os.path.join(ROOT, "include", "moco_b200.h")).read()
    body = text[text.index("typedef struct moco_resize_window"):text.index("} moco_resize_window;")]
    assert "int64_t src_offset" in body and "32 bytes" in text[text.index("} moco_resize_window;"):][:120]
    fields = [f for line in body.splitlines()[1:] if "int32_t" in line
              for f in line.split("int32_t")[1].split(";")[0].replace(" ", "").split(",")]
    assert fields == ["src_h", "src_w", "resized_h", "resized_w", "top", "left"]
    assert (A.SRC_H, A.SRC_W, A.RESIZED_H, A.RESIZED_W, A.WIN_TOP, A.WIN_LEFT, A.WIN_WORDS) == (2, 3, 4, 5, 6, 7, 8)


# --------------------------------------------------------------------------------------------------------------------
# the learning-rate schedule against the reference's

def _reference_scheduler_module():
    path = os.path.join(ROOT, "oracle", "_ref", "moco", "lr_scheduler.py")
    if not os.path.exists(path):
        pytest.skip("the reference's moco/lr_scheduler.py is not staged under oracle/_ref/")
    spec = importlib.util.spec_from_file_location("ref_lr_scheduler", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _optimizer(lrs):
    params = [torch.nn.Parameter(torch.zeros(1)) for _ in lrs]
    return torch.optim.SGD([{"params": [p], "lr": lr} for p, lr in zip(params, lrs)], lr=lrs[0], momentum=0.9)


@pytest.mark.parametrize("kind,decay", [("cosine", [30, 60, 90]), ("step", [3, 5]), ("step", [2, 4, 5])])
@pytest.mark.parametrize("warmup", [1, 2])
def test_schedule_equals_the_reference_every_iteration(kind, decay, warmup):
    import argparse
    ref_mod = _reference_scheduler_module()
    n_iter, epochs, mult, rate = 7, 6, 100, 0.1
    args = argparse.Namespace(lr_scheduler=kind, epochs=epochs, warmup_epoch=warmup, warmup_multiplier=mult,
                              lr_decay_epochs=decay, lr_decay_rate=rate)
    o_ref, o_new = _optimizer([30.0, 0.5]), _optimizer([30.0, 0.5])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref = ref_mod.get_scheduler(o_ref, n_iter, args)
        new = L.get_scheduler(o_new, n_iter, epochs, kind, warmup, mult, decay, rate)
        for t in range(epochs * n_iter + 1):
            for a, b in zip(o_ref.param_groups, o_new.param_groups):
                assert b["lr"] == pytest.approx(a["lr"], rel=1e-12, abs=0), (t, a["lr"], b["lr"])
            for o in (o_ref, o_new):
                o.step()
            ref.step()
            new.step()
    assert o_new.param_groups[0]["lr"] < 30.0


def test_schedule_without_warmup_and_bad_multiplier():
    o = _optimizer([30.0])
    s = L.get_scheduler(o, 5, 4, "cosine", 0, 100)
    assert o.param_groups[0]["lr"] == 30.0           # the reference divides by zero here
    lrs = []
    for _ in range(20):
        o.step()
        s.step()
        lrs.append(o.param_groups[0]["lr"])
    assert lrs == sorted(lrs, reverse=True) and lrs[-1] == pytest.approx(1e-6, abs=1e-12)
    o = _optimizer([30.0])
    s = L.get_scheduler(o, 5, 4, "step", 0, 100, [1, 3], 0.5)
    got = []
    for _ in range(20):
        got.append(o.param_groups[0]["lr"])
        o.step()
        s.step()
    assert got == [30.0] * 5 + [15.0] * 10 + [7.5] * 5
    with pytest.raises(ValueError, match="multiplier"):
        L.get_scheduler(_optimizer([30.0]), 5, 4, "cosine", 1, 1)
    with pytest.raises(ValueError):
        L.get_scheduler(_optimizer([30.0]), 5, 4, "poly", 1, 100)


# --------------------------------------------------------------------------------------------------------------------
# exact validation accounting across ranks

N_VAL, N_CLASS = 11, 7


def _fixed_logits():
    g = torch.Generator().manual_seed(5)
    logits = torch.randn(N_VAL, N_CLASS, generator=g)
    target = torch.randint(0, N_CLASS, (N_VAL,), generator=g)
    target[:4] = logits[:4].argmax(1)                # some top-1 hits for sure
    return logits, target


def _validate_rank(rank, world, batch=2):
    logits, target = _fixed_logits()
    ds = torch.utils.data.TensorDataset(logits, target, torch.arange(N_VAL))
    loader = torch.utils.data.DataLoader(ds, batch_size=batch, sampler=L.ShardSampler(N_VAL, rank, world))
    crit = torch.nn.CrossEntropyLoss()
    totals = torch.zeros(4, dtype=torch.float64)
    seen = []
    for out, y, idx in loader:
        totals += L.val_totals(out, y, crit(out, y))
        seen += idx.tolist()
    return L.finish_validation(totals, N_VAL), seen


def _worker(rank, world, init_file, result_dir):
    import json
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"file://{init_file}", rank=rank, world_size=world)
    try:
        res, seen = _validate_rank(rank, world)
        with open(os.path.join(result_dir, f"{rank}.json"), "w") as f:
            json.dump({"res": res, "seen": seen}, f)
    finally:
        dist.destroy_process_group()


def test_validation_totals_match_util_accuracy_at_world_1():
    (res, seen) = _validate_rank(0, 1, batch=N_VAL)
    logits, target = _fixed_logits()
    _, pred = logits.topk(5, 1, True, True)
    correct = pred.t().eq(target.view(1, -1).expand_as(pred.t()))
    assert res["n"] == N_VAL and seen == list(range(N_VAL))
    assert res["acc"] == [100.0 * float(correct[:k].reshape(-1).float().sum()) / N_VAL for k in (1, 5)]
    assert res["loss"] == pytest.approx(float(torch.nn.functional.cross_entropy(logits, target)), rel=1e-6)
    three = L.val_totals(logits[:, :3], target.clamp(max=2), torch.tensor(0.0), topk=(1, 5))
    assert float(three[2]) == N_VAL                  # top-5 of 3 classes: every sample


@pytest.mark.parametrize("world", [2, 3])
def test_validation_over_gloo_ranks_equals_world_1(tmp_path, world):
    import json
    import torch.multiprocessing as mp
    one, _ = _validate_rank(0, 1)
    mp.spawn(_worker, args=(world, str(tmp_path / "init"), str(tmp_path)), nprocs=world, join=True)
    seen = []
    for r in range(world):
        got = json.loads((tmp_path / f"{r}.json").read_text())
        assert got["res"]["n"] == N_VAL
        assert got["res"]["acc"] == one["acc"]
        assert got["res"]["loss"] == pytest.approx(one["loss"], rel=1e-6)      # fp32 batch means, other batches
        assert got["seen"] == list(range(r, N_VAL, world))
        seen += got["seen"]
    assert sorted(seen) == list(range(N_VAL))        # every index exactly once, no padding


def test_finish_validation_asserts_the_count():
    with pytest.raises(AssertionError, match="counted 10"):
        L.finish_validation(torch.tensor([1.0, 2.0, 3.0, 10.0], dtype=torch.float64), 11)


# --------------------------------------------------------------------------------------------------------------------
# the example's flags

def _example():
    spec = importlib.util.spec_from_file_location("eval_linear_example_data", os.path.join(ROOT, "examples",
                                                                                           "eval_linear.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_example_parses_the_data_flags_with_eval_py_defaults():
    mod = _example()
    a = mod.parse_args([])
    assert (a.data_dir, a.aug, a.crop, a.num_workers, a.epochs, a.lr_scheduler, a.warmup_epoch, a.warmup_multiplier,
            a.lr_decay_epochs, a.lr_decay_rate) == ("", "NULL", 0.08, 4, 100, "cosine", 5, 100, [30, 60, 90], 0.1)
    # the synthetic loop's flags keep their defaults
    assert (a.pretrained, a.model_width, a.layer, a.num_classes, a.total_batch_size, a.learning_rate, a.momentum,
            a.weight_decay, a.steps, a.val_steps, a.print_freq) == ("", 1, 6, 1000, 256, 30.0, 0.9, 0.0, 20, 2, 10)
    a = mod.parse_args(["--data-dir", "/d", "--aug", "CJ", "--crop", "0.2", "--num-workers", "8", "--epochs", "3",
                        "--lr-scheduler", "step", "--warmup-epoch", "0", "--warmup-multiplier", "10",
                        "--lr-decay-epochs", "1", "2", "--lr-decay-rate", "0.5"])
    assert (a.data_dir, a.aug, a.crop, a.num_workers, a.epochs, a.lr_scheduler, a.warmup_epoch, a.warmup_multiplier,
            a.lr_decay_epochs, a.lr_decay_rate) == ("/d", "CJ", 0.2, 8, 3, "step", 0, 10, [1, 2], 0.5)
    for bad in (["--aug", "RA"], ["--lr-scheduler", "poly"]):
        with pytest.raises(SystemExit):
            mod.parse_args(bad)
