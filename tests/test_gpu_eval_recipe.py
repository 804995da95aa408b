"""The linear evaluation's program (examples/eval_linear.py with --data-dir) on the GPU, over a seeded JPEG folder
built here, with ResNet-50 and cuDNN at torch's default settings: a run writes exactly config.json and its classifier
checkpoints; a run resumed from its first epoch's checkpoint ends with the same current.pth and the same validation,
bit for bit; -e validates that checkpoint to exactly the last epoch's figures and writes nothing; and a run without
--output-dir writes nothing."""
import gc
import importlib.util
import math
import os

import pytest
import torch
import torchvision

from moco_b200 import checkpoint

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAIN, VAL = 12, 7                    # three iterations of 4 images per epoch; a last validation batch of 3


@pytest.fixture(scope="module", autouse=True)
def _release_what_this_module_cached():
    """Hand the device memory and pinned host memory these runs left in torch's caches back to the driver, so that
    the tests after them in the same process run with the memory they would have had without them."""
    yield
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch._C._host_emptyCache()


@pytest.fixture(autouse=True)
def _default_cudnn():
    """eval_linear.py leaves cuDNN as torch starts it; other modules in the same process may not have."""
    with torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=False):
        yield


def _module():
    spec = importlib.util.spec_from_file_location("eval_linear_recipe_gpu", os.path.join(ROOT, "examples",
                                                                                         "eval_linear.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _split(root, split, n, seed0):
    g = torch.Generator().manual_seed(seed0)
    for c in range(3):
        os.makedirs(os.path.join(root, split, f"c{c}"), exist_ok=True)
    for i in range(n):
        h = int(torch.randint(60, 300, (1,), generator=g))
        w = int(torch.randint(60, 300, (1,), generator=g))
        yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
        img = torch.stack([(yy * 255) // h, (xx * 255) // w, ((yy + xx) * (3 + i % 3)) % 256]) + torch.randint(
            0, 40, (3, h, w), generator=g)
        data = torchvision.io.encode_jpeg(img.clamp(0, 255).to(torch.uint8).contiguous(), quality=90)
        with open(os.path.join(root, split, f"c{i % 3}", f"{i}.jpg"), "wb") as f:
            f.write(data.numpy().tobytes())


@pytest.fixture(scope="module")
def folder(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("eval_jpegs"))
    _split(root, "train", TRAIN, 0)
    _split(root, "val", VAL, 100)
    return root


def _argv(folder, *extra, epochs=3):
    # The encoder keeps its random initialisation, whose layer-6 features average about 20 over 2048 channels, so
    # one SGD step moves a logit by about lr * 1e6.  eval.py's learning rate of 30 is sized for a trained encoder's
    # features and would drive the loss to ~1e7 here.
    return ["--data-dir", folder, "--total-batch-size", "4", "--num-workers", "0", "--aug", "CJ", "--epochs",
            str(epochs), "--warmup-epoch", "1", "--learning-rate", "1e-7", "--save-freq", "1", "--print-freq", "1",
            *extra]


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
        assert type(a) is type(b) and a == b, what


@pytest.fixture(scope="module")
def run_a(folder, tmp_path_factory):
    """The uninterrupted three-epoch run: its output directory and what main returned."""
    with torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=False):
        out = str(tmp_path_factory.mktemp("eval_run") / "A")
        return out, _module().main(_argv(folder, "--output-dir", out))


def test_run_writes_config_and_classifier_checkpoints(run_a):
    a, res_a = run_a
    assert sorted(os.listdir(a)) == ["ckpt_epoch_1.pth", "ckpt_epoch_2.pth", "ckpt_epoch_3.pth", "config.json",
                                     "current.pth"]
    assert res_a["epoch"] == 3 and res_a["n"] == VAL and math.isfinite(res_a["loss"])
    ckpts = [checkpoint.load(os.path.join(a, f"ckpt_epoch_{i}.pth")) for i in (1, 2, 3)]
    assert res_a["best_acc1"] == max(c["best_acc1"] for c in ckpts)
    current = torch.load(os.path.join(a, "current.pth"), map_location="cpu")
    assert sorted(current) == ["best_acc1", "classifier", "epoch", "opt", "optimizer", "scheduler"]
    _assert_same(current, ckpts[2], "current")
    assert current["scheduler"] == {"last_epoch": 3 * TRAIN // 4} and len(current["optimizer"]["state"]) == 2
    w = "module.classifier.LiniearClassifier.weight"
    assert not torch.equal(ckpts[0]["classifier"][w], current["classifier"][w])


def test_resumed_run_ends_bit_identical(folder, run_a, tmp_path):
    a, res_a = run_a
    b = str(tmp_path / "B")
    res_b = _module().main(_argv(folder, "--output-dir", b, "--resume", os.path.join(a, "ckpt_epoch_1.pth")))
    assert sorted(os.listdir(b)) == ["ckpt_epoch_2.pth", "ckpt_epoch_3.pth", "config.json", "current.pth"]
    ca, cb = checkpoint.load(os.path.join(a, "current.pth")), checkpoint.load(os.path.join(b, "current.pth"))
    for key in ("classifier", "optimizer", "scheduler", "epoch", "best_acc1"):
        _assert_same(ca[key], cb[key], key)
    _assert_same(res_a, res_b, "result")


def test_evaluate_only_scores_the_checkpoint_and_writes_nothing(folder, run_a, tmp_path, monkeypatch):
    a, res_a = run_a
    monkeypatch.chdir(tmp_path)
    e = str(tmp_path / "E")
    res_e = _module().main(_argv(folder, "-e", "--resume", os.path.join(a, "current.pth"), "--output-dir", e))
    _assert_same(res_a, res_e, "result")
    assert os.listdir(tmp_path) == []


def test_run_without_output_dir_writes_nothing(folder, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    res = _module().main(_argv(folder, epochs=1))
    assert res["epoch"] == 1 and res["n"] == VAL and math.isfinite(res["loss"])
    assert os.listdir(tmp_path) == []
