"""Host side of the pre-training recipe (examples/train_moco.py with --data-dir and without --steps), no GPU needed:
the reference's command lines parse with train.py's defaults, checkpoints move both ways between this package and
the reference (staged unmodified in oracle/_ref; its pieces run in a subprocess under oracle/ref_runner.py's shims),
the learning-rate schedule survives torch.save, and an epoch's crop draws do not depend on the epochs before it."""
import argparse
import importlib.util
import json
import os
import subprocess
import sys

import pytest
import torch
import torchvision

from moco_b200 import checkpoint, encoders
from moco_b200 import linear_eval as L
from moco_b200.NCE import MemoryMoCo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")

# the pre-training command lines of the reference's README and scripts/*.sh, as the launcher hands them to train.py
README_ARGS = ["--local_rank=0", "--data-dir", "./data/imagenet", "--dataset", "imagenet", "--nce-k", "65536",
               "--output-dir", "./output/imagenet/K65536"]
SCRIPT_ARGS = ["--local_rank=0", "--data-dir", "./data/imagenet100", "--dataset", "imagenet100",
               "--base-learning-rate", "0.4", "--alpha", "0.99", "--crop", "0.08", "--nce-k", "126689", "--nce-t", "0.1",
               "--amp-opt-level", "O1", "--output-dir", "./output/imagenet100/baseLR0.4_alpha0.99_crop0.08_kall_t0.1_AMPO1"]


def _example():
    spec = importlib.util.spec_from_file_location("train_moco_example_pretrain",
                                                  os.path.join(ROOT, "examples", "train_moco.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _staged():
    if not os.path.isfile(os.path.join(REF, "train.py")):
        pytest.skip("oracle/_ref is not staged (run __graft_entry__.build() where the reference checkout exists)")


def _run_reference(code: str) -> dict:
    """Run ``code`` in a fresh interpreter with the staged reference imported as ``train`` (ref_runner's shims stay
    in that process); it prints one JSON line, which is returned."""
    prog = "import json, sys\nfrom oracle import ref_runner\ntrain = ref_runner._load_reference()\n" + code
    p = subprocess.run([sys.executable, "-c", prog], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-3000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


def test_reference_command_lines_parse_with_train_py_defaults(monkeypatch):
    _staged()
    monkeypatch.delenv("LOCAL_RANK", raising=False)
    mod = _example()
    ref = _run_reference("sys.argv = ['train.py', '--data-dir', 'd']\nprint(json.dumps(vars(train.parse_option())))")
    ours = vars(mod.parse_args(["--data-dir", "d"]))
    assert ours["steps"] is None                                  # the recipe
    ours["base_learning_rate"] = ours.pop("base_lr")
    shared = (set(ours) & set(ref)) - {"local_rank", "data_dir"}  # $LOCAL_RANK here; required there
    assert shared >= {"batch_size", "nce_k", "base_learning_rate", "epochs", "lr_scheduler", "warmup_epoch",
                      "warmup_multiplier", "lr_decay_epochs", "lr_decay_rate", "output_dir", "save_freq",
                      "print_freq", "rng_seed", "model_width", "dataset", "amp_opt_level", "crop", "aug",
                      "num_workers", "alpha", "nce_t", "momentum", "weight_decay", "resume"}
    for k in sorted(shared):
        assert ours[k] == ref[k], (k, ours[k], ref[k])

    a = mod.parse_args(README_ARGS)
    assert (a.steps, a.nce_k, a.dataset, a.output_dir, a.batch_size, a.base_lr) == (
        None, 65536, "imagenet", "./output/imagenet/K65536", 128, 0.1)
    a = mod.parse_args(SCRIPT_ARGS)
    assert (a.base_lr, a.alpha, a.crop, a.nce_k, a.nce_t, a.amp_opt_level, a.dataset) == (
        0.4, 0.99, 0.08, 126689, 0.1, "O1", "imagenet100")


def test_step_modes_keep_their_defaults(monkeypatch):
    monkeypatch.delenv("LOCAL_RANK", raising=False)
    mod = _example()
    for argv in ([], ["--data-dir", "/d", "--steps", "7"]):
        a = mod.parse_args(argv)
        assert (a.batch_size, a.nce_k, a.base_lr, a.epoch, a.save) == (256, 16384, 0.03, 1, "")
    assert mod.parse_args([]).steps == 20 and mod.parse_args(["--data-dir", "/d", "--steps", "7"]).steps == 7
    assert mod.parse_args(["--base-learning-rate", "0.5"]).base_lr == 0.5
    a = mod.parse_args(["--data-dir", "/d", "--batch-size", "64"])
    assert (a.steps, a.batch_size, a.nce_k) == (None, 64, 65536)


def _args(**kw):
    a = _example().parse_args(["--data-dir", "d"])
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _state(arch="resnet50", K=64, epoch=3):
    torch.manual_seed(0)
    model, ema = getattr(encoders, arch)(), getattr(encoders, arch)()
    contrast = MemoryMoCo(128, K, 0.07)
    opt = torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4)
    sched = L.get_scheduler(opt, 4, 10, "cosine", 1, 100)
    for _ in range(5):
        opt.step()                                                  # no gradients: only the schedule moves
        sched.step()
    return model, ema, contrast, opt, sched, checkpoint.state(_args(), epoch, model, ema, contrast, opt, sched)


def test_our_checkpoint_loads_in_the_reference_eval_and_ours(tmp_path):
    """eval.py:load_pretrained (eval.py:149-153) under torch.load's defaults, into the reference's resnet50."""
    if not os.path.isfile(os.path.join(REF, "moco", "models", "resnet.py")):
        pytest.skip("oracle/_ref is not staged")
    if REF not in sys.path:
        sys.path.insert(0, REF)
    import moco.models.resnet as ref_resnet
    model, ema, contrast, opt, sched, ckpt = _state()
    checkpoint.save(ckpt, str(tmp_path), save_freq=3)
    assert sorted(os.listdir(tmp_path)) == ["ckpt_epoch_3.pth", "current.pth"]
    path = str(tmp_path / "current.pth")

    loaded = torch.load(path, map_location="cpu")                 # weights_only=True is torch's default
    assert sorted(loaded) == ["contrast", "epoch", "model", "model_ema", "opt", "optimizer", "scheduler"]
    assert all(k.startswith("module.") for k in loaded["model"]) and loaded["epoch"] == 3
    assert loaded["scheduler"] == {"last_epoch": 5} and loaded["opt"]["nce_k"] == 65536
    ref = ref_resnet.resnet50()
    ref.load_state_dict({k.replace("module.", ""): v for k, v in loaded["model"].items()})
    ours = model.state_dict()
    for k, v in encoders.from_reference_state_dict(ref.state_dict()).items():
        assert torch.equal(v, ours[k]), k
    ref_ema = ref_resnet.resnet50()
    ref_ema.load_state_dict(loaded["model_ema"])

    # examples/eval_linear.py --pretrained
    fresh = encoders.resnet50()
    fresh.load_state_dict(encoders.from_reference_state_dict(checkpoint.load(path)["model"]))
    for k, v in fresh.state_dict().items():
        assert torch.equal(v, ours[k]), k


def test_our_checkpoint_resumes_into_our_models(tmp_path):
    model, ema, contrast, opt, sched, ckpt = _state("resnet18", K=64)
    with torch.no_grad():
        for p in model.parameters():
            p.grad = torch.randn_like(p)
    opt.step()
    ckpt = checkpoint.state(_args(), 2, model, ema, contrast, opt, sched)
    checkpoint.save(ckpt, str(tmp_path), save_freq=10)
    assert os.listdir(tmp_path) == ["current.pth"]
    torch.manual_seed(1)
    m2, e2 = encoders.resnet18(), encoders.resnet18()
    c2 = MemoryMoCo(128, 64, 0.07)
    o2 = torch.optim.SGD(m2.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4)
    assert checkpoint.restore(checkpoint.load(str(tmp_path / "current.pth")), m2, e2, c2, o2) == 3
    for a, b in ((model, m2), (ema, e2), (contrast, c2)):
        sa, sb = a.state_dict(), b.state_dict()
        assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)
    bufs = [o2.state[p]["momentum_buffer"] for p in m2.parameters()]
    assert all(torch.equal(x, opt.state[p]["momentum_buffer"]) for x, p in zip(bufs, model.parameters()))


def test_reference_checkpoint_resumes(tmp_path):
    """A current.pth written by the reference's own train.save_checkpoint (its 'opt' is an argparse.Namespace) after
    four steps over two-iteration epochs: model, model_ema, memory and every momentum buffer load, the run resumes
    at epoch 3, and the learning rate there is the reference scheduler's after those four steps."""
    _staged()
    out = str(tmp_path)
    info = _run_reference(f"""
import warnings
from oracle.ref_runner import ReferenceJob
job = ReferenceJob("resnet50", 128, 64, 0.07, batch=2, n_batches=2)
job.run(4)
args = job.args
args.output_dir, args.save_freq = {out!r}, 1
with warnings.catch_warnings():
    warnings.simplefilter("ignore")
    train.save_checkpoint(args, 2, job.model, job.model_ema, job.contrast, job.optimizer, job.scheduler)
print(json.dumps({{"lr": job.optimizer.param_groups[0]["lr"], "index": int(job.contrast.index)}}))
""")
    path = os.path.join(out, "current.pth")
    with pytest.raises(Exception):
        torch.load(path, map_location="cpu")                        # the Namespace under 'opt'
    ckpt = checkpoint.load(path)
    assert isinstance(ckpt["opt"], argparse.Namespace) and ckpt["epoch"] == 2

    args = _args(batch_size=2, nce_k=64, warmup_epoch=1)
    model, ema = encoders.resnet50(), encoders.resnet50()
    contrast = MemoryMoCo(128, 64, 0.07, persist_index=True)
    opt = torch.optim.SGD(model.parameters(), lr=args.batch_size / 256 * args.base_lr, momentum=0.9, weight_decay=1e-4)
    sched = L.get_scheduler(opt, 2, args.epochs, args.lr_scheduler, args.warmup_epoch, args.warmup_multiplier,
                            args.lr_decay_epochs, args.lr_decay_rate)
    start = checkpoint.restore(ckpt, model, ema, contrast, opt)
    sched.load_state_dict({"last_epoch": (start - 1) * 2})
    assert start == 3
    ref_model = encoders.from_reference_state_dict(ckpt["model"])
    for k, v in model.state_dict().items():
        assert torch.equal(v, ref_model[k]), k
    ref_ema = encoders.from_reference_state_dict(ckpt["model_ema"])
    for k, v in ema.state_dict().items():
        assert torch.equal(v, ref_ema[k]), k
    assert torch.equal(contrast.memory, ckpt["contrast"]["memory"])
    assert contrast.index == 0                                      # the reference never saves its ring position
    params = list(model.parameters())
    assert len(params) == 161 and len(opt.state) == 161
    for p in params:
        buf = opt.state[p]["momentum_buffer"]
        assert buf.shape == p.shape and bool(buf.abs().sum() > 0)
    assert opt.param_groups[0]["lr"] == pytest.approx(info["lr"], rel=1e-12, abs=0)
    assert info["lr"] < args.batch_size / 256 * args.base_lr       # past the warm-up, into the cosine


def test_schedule_state_survives_torch_save(tmp_path):
    for kind in ("cosine", "step"):
        o = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=0.4, momentum=0.9)
        s = L.get_scheduler(o, 3, 6, kind, 1, 100, [2, 4], 0.1)
        for _ in range(5):
            o.step()
            s.step()
        torch.save(s.state_dict(), tmp_path / "s.pth")
        expect = []
        for _ in range(10):
            o.step()
            s.step()
            expect.append(o.param_groups[0]["lr"])
        o2 = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=0.4, momentum=0.9)
        s2 = L.get_scheduler(o2, 3, 6, kind, 1, 100, [2, 4], 0.1)
        s2.load_state_dict(torch.load(tmp_path / "s.pth"))
        got = []
        for _ in range(10):
            o2.step()
            s2.step()
            got.append(o2.param_groups[0]["lr"])
        assert got == expect, kind


def _jpeg_folder(root, n=10):
    g = torch.Generator().manual_seed(3)
    for c in range(2):
        os.makedirs(os.path.join(root, "train", f"c{c}"), exist_ok=True)
    for i in range(n):
        h, w = 40 + 7 * i, 90 - 5 * i
        img = torch.randint(0, 256, (3, h, w), generator=g, dtype=torch.uint8)
        with open(os.path.join(root, "train", f"c{i % 2}", f"{i}.jpg"), "wb") as f:
            f.write(torchvision.io.encode_jpeg(img, quality=90).numpy().tobytes())


@pytest.mark.parametrize("workers", [0, 2])
def test_epoch_draws_do_not_depend_on_earlier_epochs(tmp_path, workers):
    mod = _example()
    _jpeg_folder(str(tmp_path))
    args = mod.parse_args(["--data-dir", str(tmp_path), "--batch-size", "3", "--num-workers", str(workers)])

    def epoch_records(loader, epoch):
        mod.seed_epoch(loader, args.rng_seed, epoch, 0)
        return [(params.clone(), targets.clone()) for _, params, targets in loader]

    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                             # pin_memory without a device
        ran = mod.make_recipe_loader(args, 1, 0)
        assert not ran.persistent_workers and len(ran) == 3
        e1 = epoch_records(ran, 1)
        torch.rand(5)                                               # whatever else consumed the global generator
        after = epoch_records(ran, 2)
        fresh = epoch_records(mod.make_recipe_loader(args, 1, 0), 2)
        again = epoch_records(mod.make_recipe_loader(args, 1, 0), 1)
    assert len(after) == len(fresh) == 3
    for (p, t), (q, u) in zip(after, fresh):
        assert torch.equal(p, q) and torch.equal(t, u)
    for (p, _), (q, _) in zip(e1, again):
        assert torch.equal(p, q)
    assert not all(torch.equal(p, q) for (p, _), (q, _) in zip(e1, after))
