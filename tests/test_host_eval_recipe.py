"""Host side of the linear evaluation's program (examples/eval_linear.py with --data-dir), no GPU needed: eval.py's
command lines parse with eval.py's defaults, the flags that save, resume or only validate need --data-dir, and
classifier checkpoints move both ways between this package and the reference (staged unmodified in oracle/_ref; its
pieces run in a subprocess, imported by oracle/ref_eval.py under oracle/ref_runner.py's shims)."""
import argparse
import importlib.util
import json
import os
import subprocess
import sys

import pytest
import torch

from moco_b200 import checkpoint
from moco_b200 import linear_eval as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
N_LABEL = 5

# the linear-evaluation command lines of the reference's README and scripts/*.sh, as the launcher hands them to eval.py
README_ARGS = ["--local_rank=0", "--dataset", "imagenet", "--data-dir", "./data/imagenet", "--pretrained-model",
               "./output/imagenet/K65536/current.pth", "--output-dir", "./output/imagenet/K65536/eval"]
SCRIPT_ARGS = ["--local_rank=0", "--dataset", "imagenet100", "--data-dir", "./data/imagenet100", "--pretrained-model",
               "./output/imagenet100/baseLR0.4_alpha0.99_crop0.08_kall_t0.1_AMPO1/current.pth", "--output-dir",
               "./output/imagenet100/baseLR0.4_alpha0.99_crop0.08_kall_t0.1_AMPO1/eval"]


def _example():
    spec = importlib.util.spec_from_file_location("eval_linear_example_recipe",
                                                  os.path.join(ROOT, "examples", "eval_linear.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _staged():
    if not os.path.isfile(os.path.join(REF, "eval.py")):
        pytest.skip("oracle/_ref/eval.py is not staged (run __graft_entry__.build() where the reference checkout "
                    "exists)")


def _run_reference(code: str) -> dict:
    """Run ``code`` in a fresh interpreter with the staged reference's eval.py imported as ``ev`` (ref_runner's shims
    and its one-rank gloo group stay in that process); it prints one JSON line, which is returned."""
    prog = "import json, sys\nfrom oracle import ref_eval\nev = ref_eval.load()\n" + code
    p = subprocess.run([sys.executable, "-c", prog], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-3000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


def test_reference_command_lines_parse_with_eval_py_defaults(monkeypatch):
    _staged()
    monkeypatch.delenv("LOCAL_RANK", raising=False)
    mod = _example()
    ref = _run_reference("sys.argv = ['eval.py', '--data-dir', 'd', '--pretrained-model', 'p']\n"
                         "print(json.dumps(vars(ev.parse_option())))")
    ours = vars(mod.parse_args(["--data-dir", "d", "--pretrained-model", "p"]))
    assert ours["pretrained"] == ref["pretrained_model"] == "p"
    # not compared: local_rank ($LOCAL_RANK here, None there), data_dir (required there), the pretrained model's name
    # (`pretrained` here, `pretrained_model` there) and output_dir ('' here, which writes nothing; ./output there)
    shared = (set(ours) & set(ref)) - {"local_rank", "data_dir", "output_dir"}
    assert shared >= {"dataset", "crop", "aug", "total_batch_size", "num_workers", "model", "model_width", "layer",
                      "learning_rate", "lr_scheduler", "warmup_epoch", "warmup_multiplier", "lr_decay_epochs",
                      "lr_decay_rate", "weight_decay", "momentum", "amp_opt_level", "epochs", "start_epoch", "resume",
                      "print_freq", "save_freq", "rng_seed", "eval"}
    for k in sorted(shared):
        assert ours[k] == ref[k], (k, ours[k], ref[k])
    assert ours["output_dir"] == "" and ref["output_dir"] == "./output"

    a = mod.parse_args(README_ARGS)
    assert (a.local_rank, a.dataset, a.data_dir, a.pretrained, a.output_dir, a.model, a.amp_opt_level) == (
        0, "imagenet", "./data/imagenet", "./output/imagenet/K65536/current.pth", "./output/imagenet/K65536/eval",
        "resnet50", "O0")
    a = mod.parse_args(SCRIPT_ARGS)
    assert (a.dataset, a.data_dir, a.output_dir, a.epochs, a.start_epoch, a.eval) == (
        "imagenet100", "./data/imagenet100", "./output/imagenet100/baseLR0.4_alpha0.99_crop0.08_kall_t0.1_AMPO1/eval",
        100, 1, False)


def test_program_flags_need_data_dir(monkeypatch):
    monkeypatch.delenv("LOCAL_RANK", raising=False)
    mod = _example()
    for flags in (["--resume", "c.pth"], ["-e"], ["--eval"], ["--output-dir", "out"], ["--start-epoch", "2"]):
        with pytest.raises(SystemExit):
            mod.parse_args(flags)
        a = mod.parse_args(["--data-dir", "d", *flags])
        assert a.data_dir == "d"
    for bad in (["--data-dir", "d", "--start-epoch", "0"], ["--dataset", "cifar"], ["--model", "resnet18"],
                ["--amp-opt-level", "O3"]):
        with pytest.raises(SystemExit):
            mod.parse_args(bad)
    a = mod.parse_args([])                              # the synthetic loop: the new flags at their defaults
    assert (a.output_dir, a.resume, a.eval, a.start_epoch, a.save_freq, a.rng_seed) == ("", "", False, 1, 5, 0)


def _args(**kw):
    a = _example().parse_args(["--data-dir", "d"])
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _trained(layer=6, n_label=N_LABEL, steps=5, n_iter=2):
    """Our classifier, SGD and schedule after ``steps`` steps on random features."""
    torch.manual_seed(0)
    clf = L.LinearClassifierResNet(layer, n_label)
    opt = torch.optim.SGD(clf.parameters(), lr=30.0, momentum=0.9)
    sched = L.get_scheduler(opt, n_iter, 10, "cosine", 1, 100)
    g = torch.Generator().manual_seed(1)
    for _ in range(steps):
        x, y = torch.randn(4, 2048, generator=g), torch.randint(0, n_label, (4,), generator=g)
        loss = torch.nn.functional.cross_entropy(clf(x), y)
        opt.zero_grad()
        loss.backward()
        opt.step()
        sched.step()
    return clf, opt, sched


def test_our_classifier_checkpoint_has_eval_py_keys_and_loads_in_the_reference(tmp_path):
    clf, opt, sched = _trained()
    ckpt = checkpoint.classifier_state(_args(), 3, clf, torch.tensor(41.5), opt, sched)
    checkpoint.save(ckpt, str(tmp_path), save_freq=3)
    assert sorted(os.listdir(tmp_path)) == ["ckpt_epoch_3.pth", "current.pth"]
    path = str(tmp_path / "current.pth")
    loaded = torch.load(path, map_location="cpu")                 # weights_only=True is torch's default
    assert sorted(loaded) == ["best_acc1", "classifier", "epoch", "opt", "optimizer", "scheduler"]
    assert loaded["epoch"] == 3 and loaded["scheduler"] == {"last_epoch": 5}
    assert type(loaded["best_acc1"]) is float and loaded["best_acc1"] == 41.5
    assert loaded["opt"]["save_freq"] == 5 and loaded["opt"]["data_dir"] == "d"
    assert list(loaded["classifier"]) == ["module." + k for k in clf.state_dict()]
    for k, v in clf.state_dict().items():
        assert torch.equal(loaded["classifier"]["module." + k], v), k
    assert len(loaded["optimizer"]["state"]) == 2

    _staged()
    got = _run_reference(f"""
import torch
from torch.nn.parallel import DistributedDataParallel
from moco.models.LinearModel import LinearClassifierResNet
ckpt = torch.load({path!r}, map_location="cpu")
clf = DistributedDataParallel(LinearClassifierResNet(6, {N_LABEL}, "avg", 1), broadcast_buffers=False)   # eval.py:211
clf.load_state_dict(ckpt["classifier"])
sd = clf.state_dict()
print(json.dumps({{"keys": list(sd), "equal": all(torch.equal(v, ckpt["classifier"][k]) for k, v in sd.items())}}))
""")
    assert got["keys"] == list(loaded["classifier"]) and got["equal"]


def test_reference_classifier_checkpoint_restores(tmp_path):
    """A checkpoint written by the reference's own eval.save_checkpoint (its 'opt' is an argparse.Namespace, its
    'best_acc1' a tensor) after four SGD steps over two-iteration epochs under its get_scheduler: the classifier
    and every momentum buffer load, the run resumes at epoch 3 with the reference's best_acc1, and the learning rate
    there is the reference scheduler's after those four steps."""
    _staged()
    out = str(tmp_path)
    info = _run_reference(f"""
import warnings
import torch
from torch.nn.parallel import DistributedDataParallel
from moco.lr_scheduler import get_scheduler
from moco.models.LinearModel import LinearClassifierResNet
sys.argv = ["eval.py", "--data-dir", "d", "--pretrained-model", "p", "--output-dir", {out!r}, "--warmup-epoch", "1",
            "--epochs", "10"]
args = ev.parse_option()
clf = LinearClassifierResNet(args.layer, {N_LABEL}, "avg", args.model_width)                       # eval.py:145
opt = torch.optim.SGD(clf.parameters(), lr=args.learning_rate, momentum=args.momentum,
                      weight_decay=args.weight_decay)                                              # eval.py:196-199
sched = get_scheduler(opt, 2, args)
clf = DistributedDataParallel(clf, broadcast_buffers=False)                                        # eval.py:211
g = torch.Generator().manual_seed(2)
with warnings.catch_warnings():
    warnings.simplefilter("ignore")
    for _ in range(4):
        x, y = torch.randn(4, 2048, generator=g), torch.randint(0, {N_LABEL}, (4,), generator=g)
        loss = torch.nn.functional.cross_entropy(clf(x), y)
        opt.zero_grad()
        loss.backward()
        opt.step()
        sched.step()
    ev.save_checkpoint(args, 2, clf, torch.tensor(37.5), opt, sched)
print(json.dumps({{"lr": opt.param_groups[0]["lr"]}}))
""")
    assert sorted(os.listdir(out)) == ["ckpt_epoch_2.pth", "current.pth"]
    path = os.path.join(out, "current.pth")
    with pytest.raises(Exception):
        torch.load(path, map_location="cpu")                        # the Namespace under 'opt'
    ckpt = checkpoint.load(path)
    assert isinstance(ckpt["opt"], argparse.Namespace) and ckpt["epoch"] == 2
    assert isinstance(ckpt["best_acc1"], torch.Tensor)

    args = _args(warmup_epoch=1, epochs=10)
    clf = L.LinearClassifierResNet(args.layer, N_LABEL, "avg", args.model_width)
    opt = torch.optim.SGD(clf.parameters(), lr=args.learning_rate, momentum=args.momentum,
                          weight_decay=args.weight_decay)
    sched = L.get_scheduler(opt, 2, args.epochs, args.lr_scheduler, args.warmup_epoch, args.warmup_multiplier,
                            args.lr_decay_epochs, args.lr_decay_rate)
    start, best = checkpoint.restore_classifier(ckpt, clf, opt)
    sched.load_state_dict({"last_epoch": (start - 1) * 2})
    assert (start, best) == (3, 37.5) and type(best) is float
    ref_sd = ckpt["classifier"]
    assert all(k.startswith("module.") for k in ref_sd)
    for k, v in clf.state_dict().items():
        assert torch.equal(v, ref_sd["module." + k]), k
    params = list(clf.parameters())
    assert len(params) == 2 and len(opt.state) == 2
    for i, p in enumerate(params):
        buf = opt.state[p]["momentum_buffer"]
        assert torch.equal(buf, ckpt["optimizer"]["state"][i]["momentum_buffer"]) and bool(buf.abs().sum() > 0)
    assert opt.param_groups[0]["lr"] == pytest.approx(info["lr"], rel=1e-12, abs=0)
    assert info["lr"] < args.learning_rate                          # past the warm-up, into the cosine


def test_restore_without_the_module_prefix():
    clf, opt, sched = _trained()
    ckpt = checkpoint.classifier_state(_args(), 4, clf, 12.0, opt, sched)
    ckpt["classifier"] = {k.removeprefix("module."): v for k, v in ckpt["classifier"].items()}
    c2 = L.LinearClassifierResNet(6, N_LABEL)
    o2 = torch.optim.SGD(c2.parameters(), lr=30.0, momentum=0.9)
    assert checkpoint.restore_classifier(ckpt, c2, o2) == (5, 12.0)
    for k, v in clf.state_dict().items():
        assert torch.equal(v, c2.state_dict()[k]), k


@pytest.mark.parametrize("layer,n_label,width", [(6, N_LABEL + 1, 1), (5, N_LABEL, 1), (4, N_LABEL, 1),
                                                 (6, N_LABEL, 2)])
def test_restore_into_another_classifier_raises(layer, n_label, width):
    clf, opt, sched = _trained()
    ckpt = checkpoint.classifier_state(_args(), 1, clf, 0.0, opt, sched)
    other = L.LinearClassifierResNet(layer, n_label, "avg", width)
    with pytest.raises(RuntimeError, match="size mismatch"):
        checkpoint.restore_classifier(ckpt, other, torch.optim.SGD(other.parameters(), lr=30.0, momentum=0.9))
