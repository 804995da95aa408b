"""The frozen-BatchNorm path of the linear evaluation: moco_bn_eval_act, moco_bn_relu_maxpool_eval and
moco_bn_eval_act_avgpool against the header's numerical contract written as separate fp32 torch ops (bit for bit), a
whole frozen ResNet against a module-by-module oracle built from the same convolutions (bit for bit) and against the
reference's fp32 model, the opt-in rules, and examples/eval_linear.py."""
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EVAL_KERNELS = ("moco_bn_eval_act", "moco_bn_relu_maxpool_eval", "moco_bn_eval_act_avgpool")


def _cl(t):
    return t.bfloat16().contiguous(memory_format=torch.channels_last)


def _coefs(C, dev, g):
    s = torch.rand(C, device=dev, generator=g) + 0.5
    t = torch.randn(C, device=dev, generator=g) * 0.3
    s[1], t[1] = 1e-42, 0.0             # outputs that underflow to zero in bf16
    t[2] = -1e4                         # exact ReLU zeros over a whole channel
    return s, t


def _bc(v):
    return v.view(1, -1, 1, 1)


def _contract(x, s, t, r=None, s2=None, t2=None, relu=True):
    """include/moco_b200.h's eval contract as separate fp32 torch ops (no FMA)."""
    z = x.float() * _bc(s) + _bc(t)
    if r is not None:
        rr = r.float() if s2 is None else (r.float() * _bc(s2) + _bc(t2)).bfloat16().float()
        z = z + rr
    if relu:
        z = z.relu()
    return z.bfloat16()


def _avgpool(y):
    """Per-pixel fp32 accumulation in increasing pixel order, one division."""
    N, C, H, W = y.shape
    flat = y.float().reshape(N, C, H * W)
    acc = torch.zeros(N, C, dtype=torch.float32, device=y.device)
    for p in range(H * W):
        acc = acc + flat[:, :, p]
    return acc / torch.full_like(acc, H * W)


def _ptr(t):
    return t.data_ptr() if t is not None else None


# C in {64, 256, 2048}; M = N * H * W not a multiple of 32; HW = 49 and HW = 15 (not a multiple of 8)
SHAPES = [(5, 64, 9, 9), (3, 256, 7, 7), (2, 2048, 7, 5), (3, 2048, 7, 7), (4, 256, 5, 3)]
CASES = [("none", True), ("none", False), ("identity", True), ("identity", False), ("shortcut", True)]


@pytest.mark.parametrize("N,C,H,W", SHAPES)
@pytest.mark.parametrize("res,relu", CASES)
def test_eval_act_and_avgpool_match_the_contract(N, C, H, W, res, relu):
    from moco_b200 import _lib
    lib = _lib.load()
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(N * C + H * 3 + W)
    s, t = _coefs(C, dev, g)
    x = _cl(torch.randn((N, C, H, W), device=dev, generator=g) * 1.5 + 0.2)
    r = s2 = t2 = None
    if res != "none":
        r = torch.randn((N, C, H, W), device=dev, generator=g)
        r[:, 1] = 0.0
        r = _cl(r)
    if res == "shortcut":
        s2, t2 = torch.rand(C, device=dev, generator=g) + 0.5, torch.randn(C, device=dev, generator=g) * 0.3
        t2[1] = 0.0                     # keeps the underflow channel at zero
    want = _contract(x, s, t, r, s2, t2, relu)
    y = torch.empty_like(x)
    st = _lib.cur_stream()
    assert lib.moco_bn_eval_act(x.data_ptr(), _ptr(r), y.data_ptr(), N * H * W, C, s.data_ptr(), t.data_ptr(),
                                int(relu), _ptr(s2), _ptr(t2), st) == 0
    feat = torch.empty((N, C), dtype=torch.float32, device=dev)
    assert lib.moco_bn_eval_act_avgpool(x.data_ptr(), _ptr(r), feat.data_ptr(), N, H * W, C, s.data_ptr(),
                                        t.data_ptr(), int(relu), _ptr(s2), _ptr(t2), st) == 0
    torch.cuda.synchronize()
    assert torch.equal(y, want)
    assert torch.equal(feat, _avgpool(want))
    assert bool((y[:, 1] == 0).all())
    if relu:
        assert bool((y == 0).any()) and bool((y > 0).any())


# odd and even H / W; C = 64 (the stem) and 256
POOL_SHAPES = [(4, 64, 112, 112), (3, 64, 9, 11), (2, 256, 7, 6), (5, 64, 1, 3)]


@pytest.mark.parametrize("N,C,H,W", POOL_SHAPES)
def test_stem_eval_maxpool_matches_the_contract(N, C, H, W):
    from moco_b200 import _lib
    lib = _lib.load()
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(N * 100 + H * 7 + W)
    s, t = _coefs(C, dev, g)
    x = _cl(torch.randint(-3, 4, (N, C, H, W), device=dev, generator=g).float() * 0.5)      # many pool ties
    want = F.max_pool2d(_contract(x, s, t), 3, 2, 1)
    y = torch.empty_like(want).contiguous(memory_format=torch.channels_last)
    assert lib.moco_bn_relu_maxpool_eval(x.data_ptr(), y.data_ptr(), N, H, W, C, s.data_ptr(), t.data_ptr(),
                                         _lib.cur_stream()) == 0
    torch.cuda.synchronize()
    assert torch.equal(y, want)


def _randomise(model, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                C = m.num_features
                m.weight.copy_(torch.rand(C, generator=g) + 0.5)
                m.bias.copy_(torch.randn(C, generator=g) * 0.2)
                m.running_mean.copy_(torch.randn(C, generator=g) * 0.3)
                m.running_var.copy_(torch.rand(C, generator=g) + 0.5)


def _fold(bn):
    s = bn.weight / torch.sqrt(bn.running_var + bn.eps)
    return s, bn.bias - bn.running_mean * s


def _oracle(m, x, layer):
    """The frozen forward module by module: the model's own convolutions and the contract's torch ops."""
    from moco_b200 import encoders
    from moco_b200.util import crop_to_s2d_bf16
    if layer <= 0:
        return x

    def bn(mod, z, r=None, sc=None):
        s, t = _fold(mod)
        s2, t2 = _fold(sc) if sc is not None else (None, None)
        return _contract(z, s, t, r, s2, t2, mod.relu)

    x = F.max_pool2d(bn(m.stem[1], m.stem[0](crop_to_s2d_bf16(x))), 3, 2, 1)
    if layer == 1:
        return x
    ends = [sum(m.depths[:i + 1]) for i in range(len(m.depths))]
    for i, b in enumerate(m.layers):
        y = bn(b.bn1, b.conv1(x))
        if isinstance(b, encoders._Bottleneck):
            y = bn(b.bn2, b.conv2(y))
            last, conv = b.bn3, b.conv3
        else:
            last, conv = b.bn2, b.conv2
        x = bn(last, conv(y), x if b.short is None else b.short[0](x), None if b.short is None else b.short[1])
        if i + 1 in ends and layer == 2 + ends.index(i + 1):
            return x
    x = _avgpool(x)
    if layer == 6:
        return x
    x = m.fc(x).float()
    return x / x.pow(2).sum(1, keepdim=True).sqrt()


@pytest.fixture
def deterministic_cudnn():
    b, d = torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    yield
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = b, d


@pytest.mark.parametrize("arch", ["resnet50", "resnet18"])
def test_frozen_encoder_equals_the_contract_module_by_module(arch, deterministic_cudnn):
    from moco_b200 import encoders, _lib
    dev = torch.device("cuda:0")
    torch.manual_seed(5)
    m = getattr(encoders, arch)(128).to(memory_format=torch.channels_last)
    _randomise(m, 6)
    m = m.to(dev).freeze()
    x = torch.randn(4, 3, 224, 224, device=dev)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for layer in range(1, 8):
            before = _lib.launches
            got = m(x, layer)
            launched = _lib.launches - before
            n_bn = sum(1 for b in m.layers) * (3 if arch == "resnet50" else 2)
            want = _oracle(m, x, layer)
            assert got.dtype == want.dtype and got.shape == want.shape, layer
            assert torch.equal(got, want), layer
            if layer == 7:
                # input pass + stem + every block's BatchNorms (shortcut BNs folded in): one launch each
                assert launched == 1 + 1 + n_bn, launched
        assert got.shape == (4, 128)


def test_frozen_features_are_close_to_the_reference_fp32_model(deterministic_cudnn):
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isfile(os.path.join(ref_dir, "moco", "models", "resnet.py")):
        pytest.skip("oracle/_ref is not staged (run __graft_entry__.build() where the reference checkout exists)")
    if ref_dir not in sys.path:
        sys.path.insert(0, ref_dir)
    from moco.models.resnet import resnet50 as ref_resnet50
    from moco_b200 import encoders
    dev = torch.device("cuda:0")
    torch.manual_seed(8)
    theirs = ref_resnet50()
    _randomise(theirs, 9)
    theirs = theirs.to(dev).eval()
    ours = encoders.resnet50().to(memory_format=torch.channels_last)
    ours.load_state_dict(encoders.from_reference_state_dict(theirs.state_dict()))
    ours = ours.to(dev).freeze()
    x = torch.randn(8, 3, 224, 224, device=dev)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            for layer in range(1, 8):
                want = theirs(x, layer).float()
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    got = ours(x, layer).float()
                rel = float((got - want).norm() / want.norm())
                print(f"layer {layer}: relative L2 error of the frozen bf16 path against fp32 = {rel:.3e}")
                # bf16 activations and weights (8 significant bits): a few 1e-3 per layer, compounding over the depth
                assert rel < 5e-2, (layer, rel)
    finally:
        torch.backends.cudnn.allow_tf32 = prev


@pytest.fixture
def spy(monkeypatch):
    from moco_b200 import _lib
    lib = _lib.load()
    calls = []
    for name in EVAL_KERNELS:
        orig = getattr(lib, name)
        monkeypatch.setattr(lib, name, lambda *a, _o=orig, _n=name: (calls.append(_n), _o(*a))[1])
    return calls


def _pair(arch="resnet18"):
    from moco_b200 import encoders
    dev = torch.device("cuda:0")
    torch.manual_seed(1)
    a = getattr(encoders, arch)(128).to(memory_format=torch.channels_last)
    _randomise(a, 2)
    b = getattr(encoders, arch)(128).to(memory_format=torch.channels_last)
    b.load_state_dict(a.state_dict())
    return a.to(dev), b.to(dev)


def test_unfrozen_eval_launches_none_of_the_eval_kernels(spy):
    from moco_b200.util import crop_to_s2d_bf16
    plain, _ = _pair()
    plain.eval()
    x = crop_to_s2d_bf16(torch.randn(2, 3, 64, 64, device="cuda"))
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        for layer in (1, 5, 6, 7):
            plain(x, layer)
    assert spy == []


def test_frozen_model_in_train_or_with_grad_takes_the_unfrozen_path(spy, deterministic_cudnn):
    from moco_b200.util import crop_to_s2d_bf16
    plain, frozen = _pair()
    frozen.freeze()
    x = crop_to_s2d_bf16(torch.randn(4, 3, 64, 64, device="cuda"))
    plain.eval()
    with torch.autocast("cuda", dtype=torch.bfloat16):           # grad mode on
        assert torch.equal(frozen(x, 6), plain(x, 6))
    assert spy == []
    plain.train()
    frozen.train()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        assert torch.equal(frozen(x, 7), plain(x, 7))
    for (n, p), (_, q) in zip(frozen.named_buffers(), plain.named_buffers()):
        assert torch.equal(p, q), n                               # the same running-statistics updates
    assert spy == []
    frozen.eval()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        frozen(x, 6)
    assert set(spy) == set(EVAL_KERNELS)


@pytest.mark.parametrize("memory_format", [torch.contiguous_format, torch.channels_last])
def test_frozen_fp32_model_without_autocast_runs_the_unfrozen_path(spy, deterministic_cudnn, memory_format):
    """eval.py's default (--amp-opt-level O0): fp32 weights and images, no autocast.  The stem keeps its fp32 7x7
    convolution (no space-to-depth bf16 input) and every BatchNorm runs nn.BatchNorm2d, as for an unfrozen model."""
    plain, frozen = _pair()
    plain, frozen = plain.to(memory_format=memory_format).eval(), frozen.to(memory_format=memory_format).freeze()
    x = torch.randn(2, 3, 64, 64, device="cuda").contiguous(memory_format=memory_format)
    with torch.no_grad():
        for layer in (1, 3, 5, 6, 7):
            got = frozen(x, layer)
            assert got.dtype == torch.float32, layer
            assert torch.equal(got, plain(x, layer)), layer
    assert spy == []


def test_set_fused_false_keeps_a_frozen_model_on_the_torch_ops(spy, deterministic_cudnn):
    from moco_b200 import bn
    plain, frozen = _pair()
    plain.eval()
    frozen.freeze()
    x = torch.randn(2, 3, 64, 64, device="cuda")
    bn.set_fused(False)
    try:
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            for layer in (1, 5, 6, 7):
                assert torch.equal(frozen(x, layer), plain(x, layer)), layer
    finally:
        bn.set_fused(True)
    assert spy == []


def test_freeze_again_drops_coefficients_written_through_data(deterministic_cudnn):
    a, b = _pair()
    a.freeze()
    b.freeze()
    x = torch.randn(2, 3, 64, 64, device="cuda")
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        before = a(x, 6)
        for m in (a, b):
            m.stem[1].running_var.data.mul_(4.0)           # .data: the version counter does not move
        a.freeze()
        assert not torch.equal(a(x, 6), before)
        assert torch.equal(a(x, 6), b.freeze()(x, 6))


def test_load_state_dict_after_freeze_refolds(spy, deterministic_cudnn):
    a, b = _pair()
    a.freeze()
    b.freeze()
    other = {k: v.clone() for k, v in b.state_dict().items()}
    for k in other:
        if k.endswith("running_var"):
            other[k] *= 2.0
        elif k.endswith("bias") and "fc" not in k:
            other[k] += 0.1
    x = torch.randn(2, 3, 64, 64, device="cuda")
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        before = a(x, 6)
        a.load_state_dict(other)
        after = a(x, 6)
        b.load_state_dict(other)
        fresh = b(x, 6)
    assert not torch.equal(before, after)
    assert torch.equal(after, fresh)
    assert spy


def test_eval_linear_example_runs_from_both_checkpoint_namings(tmp_path):
    from moco_b200.encoders import to_reference_state_dict
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    ours = str(tmp_path / "moco.pth")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "train_moco.py"), "--arch", "resnet50",
                        "--batch-size", "8", "--nce-k", "256", "--steps", "2", "--save", ours],
                       capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
    assert p.returncode == 0, p.stderr[-3000:]
    ckpt = torch.load(ours, map_location="cpu")
    assert ckpt["epoch"] == 1
    theirs = str(tmp_path / "reference_keys.pth")
    torch.save({"model": {"module." + k: v for k, v in to_reference_state_dict(ckpt["model"]).items()},
                "epoch": ckpt["epoch"]}, theirs)
    for path in (ours, theirs):
        p = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "eval_linear.py"), "--pretrained", path,
                            "--steps", "3", "--val-steps", "1", "--total-batch-size", "16", "--num-classes", "10",
                            "--print-freq", "1"], capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
        assert p.returncode == 0, p.stderr[-3000:]
        losses = [float(v) for v in re.findall(r"loss (\S+)", p.stdout)]
        assert len(losses) == 4 and all(v == v and abs(v) < float("inf") for v in losses), p.stdout
