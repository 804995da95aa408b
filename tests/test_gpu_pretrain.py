"""The pre-training recipe (examples/train_moco.py with --data-dir and without --steps) on the GPU, over a seeded JPEG
folder built here: a run resumed from an epoch checkpoint ends bit-identical to the uninterrupted run, with and
without the fused-normalize / graphed tail; without --persist-index the resumed ring restarts at slot 0 as in the
reference; the pixel prefetch feeds the steps exactly what a plain loop over the same loader does; and the
checkpoint it writes is evaluated by examples/eval_linear.py."""
import gc
import importlib.util
import math
import os

import pytest
import torch
import torchvision

from moco_b200 import checkpoint
from moco_b200 import train_step

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BATCH, K, IMAGES = 8, 64, 24          # three iterations per epoch; 24 keys per epoch wrap the 64-slot ring


@pytest.fixture(scope="module", autouse=True)
def _release_what_this_module_cached():
    """Hand the device memory and pinned host memory these runs left in torch's caches back to the driver, so that
    the tests after them in the same process run with the memory they would have had without them."""
    yield
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch._C._host_emptyCache()


def _module(name, path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "examples", path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _split(root, split, n, seed0):
    g = torch.Generator().manual_seed(seed0)
    for c in range(3):
        os.makedirs(os.path.join(root, split, f"c{c}"), exist_ok=True)
    for i in range(n):
        h = int(torch.randint(60, 200, (1,), generator=g))
        w = int(torch.randint(60, 200, (1,), generator=g))
        yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
        img = torch.stack([(yy * 255) // h, (xx * 255) // w, ((yy + xx) * 5) % 256]) + torch.randint(0, 40, (3, h, w),
                                                                                                       generator=g)
        data = torchvision.io.encode_jpeg(img.clamp(0, 255).to(torch.uint8).contiguous(), quality=90)
        with open(os.path.join(root, split, f"c{i % 3}", f"{i}.jpg"), "wb") as f:
            f.write(data.numpy().tobytes())


@pytest.fixture(scope="module")
def folder(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("pretrain_jpegs"))
    _split(root, "train", IMAGES, 0)
    _split(root, "val", 7, 100)
    return root


def _recipe(folder, out, *extra, arch="resnet18", epochs=3):
    return ["--data-dir", folder, "--arch", arch, "--batch-size", str(BATCH), "--nce-k", str(K), "--epochs",
            str(epochs), "--warmup-epoch", "1", "--save-freq", "1", "--num-workers", "0", "--print-freq", "1",
            "--output-dir", out, *extra]


def _assert_same(a, b, what=""):
    if isinstance(a, dict):
        assert list(a) == list(b), what
        for k in a:
            _assert_same(a[k], b[k], f"{what}.{k}")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            _assert_same(x, y, f"{what}[{i}]")
    elif isinstance(a, torch.Tensor):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), what
    else:
        assert a == b, what


@pytest.mark.parametrize("fused", [False, True], ids=["plain", "fused_graph"])
def test_resumed_run_ends_bit_identical(folder, tmp_path, fused):
    mod = _module("train_moco_pretrain_gpu", "train_moco.py")
    flags = ["--persist-index"] + (["--fuse-normalize", "--graph-tail"] if fused else [])
    a, b = str(tmp_path / "A"), str(tmp_path / "B")
    mod.main(_recipe(folder, a, *flags))
    assert sorted(os.listdir(a)) == ["ckpt_epoch_1.pth", "ckpt_epoch_2.pth", "ckpt_epoch_3.pth", "config.json",
                                     "current.pth"]
    mod.main(_recipe(folder, b, *flags, "--resume", os.path.join(a, "ckpt_epoch_1.pth")))
    ca, cb = checkpoint.load(os.path.join(a, "current.pth")), checkpoint.load(os.path.join(b, "current.pth"))
    assert ca["epoch"] == cb["epoch"] == 3
    assert int(ca["contrast"]["params"]) == (3 * IMAGES) % K
    for key in ("model", "model_ema", "contrast", "optimizer", "scheduler"):
        _assert_same(ca[key], cb[key], key)
    assert len(ca["optimizer"]["state"]) == 62                      # a momentum buffer for every ResNet-18 parameter
    first = checkpoint.load(os.path.join(a, "ckpt_epoch_1.pth"))
    assert not torch.equal(first["model"]["module.fc.weight"], ca["model"]["module.fc.weight"])


def test_resume_without_persist_index_restarts_the_ring(folder, tmp_path):
    """The reference never saves its ring position: the resumed run writes its 48 keys to slots 0..47 and leaves
    the checkpoint's slots 48..63 alone, where the uninterrupted run continued at slot 24 and wrapped."""
    mod = _module("train_moco_pretrain_gpu_ring", "train_moco.py")
    a, b = str(tmp_path / "A"), str(tmp_path / "B")
    mod.main(_recipe(folder, a))
    mod.main(_recipe(folder, b, "--resume", os.path.join(a, "ckpt_epoch_1.pth")))
    m1 = checkpoint.load(os.path.join(a, "ckpt_epoch_1.pth"))["contrast"]["memory"]
    ma = checkpoint.load(os.path.join(a, "current.pth"))["contrast"]["memory"]
    mb = checkpoint.load(os.path.join(b, "current.pth"))["contrast"]["memory"]
    written = 2 * IMAGES
    assert torch.equal(mb[written:], m1[written:])
    assert not torch.equal(ma[written:], m1[written:])
    assert all(not torch.equal(mb[i], m1[i]) for i in range(written))


def test_prefetch_feeds_the_steps_what_a_plain_loop_does(folder, tmp_path, monkeypatch):
    from moco_b200 import encoders
    from moco_b200.augment import augment_two_crop
    from moco_b200.linear_eval import get_scheduler
    from moco_b200.NCE import MemoryMoCo
    from moco_b200.util import moment_update
    mod = _module("train_moco_pretrain_gpu_prefetch", "train_moco.py")
    losses = []
    call = train_step.MoCoStep.__call__

    def recording(self, x1, x2, epoch):
        loss, prob = call(self, x1, x2, epoch)
        losses.append((loss.detach().clone(), prob.detach().clone()))
        return loss, prob
    monkeypatch.setattr(train_step.MoCoStep, "__call__", recording)
    argv = _recipe(folder, str(tmp_path / "A"), epochs=2)
    mod.main(argv)
    recipe = [(float(l), float(p)) for l, p in losses]
    assert len(recipe) == 2 * IMAGES // BATCH
    losses.clear()

    # the same recipe written out by hand, with the pixels copied by augment_two_crop on the compute stream
    args = mod.parse_args(argv)
    dev = torch.device("cuda", 0)
    loader = mod.make_recipe_loader(args, 1, 0)
    torch.manual_seed(args.rng_seed)
    model = encoders.resnet18(low_dim=128).to(dev).to(memory_format=torch.channels_last)
    ema = encoders.resnet18(low_dim=128).to(dev).to(memory_format=torch.channels_last)
    moment_update(model, ema, 0)
    contrast = MemoryMoCo(128, K, args.nce_t).to(dev)
    opt = torch.optim.SGD(model.parameters(), lr=BATCH / 256 * args.base_lr, momentum=0.9, weight_decay=1e-4)
    sched = get_scheduler(opt, len(loader), args.epochs, "cosine", 1, 100)
    step = train_step.MoCoStep(model, ema, contrast, opt, channels_last=True)
    for epoch in (1, 2):
        mod.seed_epoch(loader, args.rng_seed, epoch, 0)
        for batch in loader:
            x1, x2 = torch.split(augment_two_crop(batch), [3, 3], dim=1)
            step(x1, x2, epoch)
            sched.step()
    plain = [(float(l), float(p)) for l, p in losses]
    assert recipe == plain
    assert all(math.isfinite(l) for l, _ in recipe)


def test_pretrain_then_evaluate(folder, tmp_path):
    train = _module("train_moco_pretrain_gpu_r50", "train_moco.py")
    out = str(tmp_path / "R50")
    res = train.main(_recipe(folder, out, arch="resnet50", epochs=1))
    assert res["epoch"] == 1 and math.isfinite(res["loss"])
    ev = _module("eval_linear_pretrain_gpu", "eval_linear.py")
    got = ev.main(["--pretrained", os.path.join(out, "current.pth"), "--data-dir", folder, "--epochs", "1",
                   "--total-batch-size", "4", "--num-workers", "0"])
    assert got["n"] == 7 and math.isfinite(got["loss"])
