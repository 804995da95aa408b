"""moco_conv1x1_bn_stats (csrc/conv1x1_sm90.cu): the 1x1 convolution forward with the next BatchNorm's batch
statistics, at every stride-1 1x1 shape of ResNet-50's bottleneck blocks; moco_bn_fwd_train_given; and the encoder
wiring of bn.conv1x1_stats against the same model on cuDNN's convolutions and the statistics passes."""
import math

import pytest
import torch
import torch.nn.functional as F
from torch.utils._python_dispatch import TorchDispatchMode

pytestmark = pytest.mark.gpu

# (side at batch 256, Cin, Cout) of ResNet-50's stride-1 1x1 convolutions
SHAPES = [(56, 64, 64), (56, 256, 64), (56, 64, 256), (56, 256, 128), (28, 512, 128), (28, 128, 512),
          (28, 512, 256), (14, 1024, 256), (14, 256, 1024), (14, 1024, 512), (7, 2048, 512), (7, 512, 2048)]
# reduced batches for the exact-arithmetic cases: M = N * side^2 is not a multiple of the 128-row tile for most
SMALL_N = {56: 2, 28: 3, 14: 5, 7: 3}


def _cl(t):
    return t.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)


def _f32(C, dev):
    return torch.empty(C, dtype=torch.float32, device=dev)


def _run(x, w, stats, momentum=0.1, eps=1e-5):
    """moco_conv1x1_bn_stats -> (y, mean, invstd); stats = (running_mean, running_var, num_batches_tracked) or None."""
    from moco_b200 import _lib
    from moco_b200.bn import _layer, _workspace
    lib = _lib.load()
    N, Cin, H, W = x.shape
    Cout = w.shape[0]
    y = torch.empty((N, Cout, H, W), dtype=torch.bfloat16, device=x.device, memory_format=torch.channels_last)
    mean, invstd = _f32(Cout, x.device), _f32(Cout, x.device)
    rm, rv, nbt = stats if stats is not None else (None, None, None)
    ws = _workspace(x.device, conv=True)
    before = _lib.launches
    _lib.check(lib.moco_conv1x1_bn_stats(x.data_ptr(), w.data_ptr(), y.data_ptr(), N * H * W, Cin, Cout,
                                         _layer(None, None, mean, invstd, (rm, rv, nbt, momentum, eps)),
                                         ws.data_ptr(), ws.numel(), _lib.cur_stream()), "moco_conv1x1_bn_stats")
    assert _lib.launches == before + 1
    return y, mean, invstd


def _bn_stats_of(y, stats, momentum=0.1, eps=1e-5):
    """moco_bn_fwd_train's statistics of y (its output discarded)."""
    from moco_b200 import _lib
    from moco_b200.bn import _workspace
    lib = _lib.load()
    N, C, H, W = y.shape
    mean, invstd = _f32(C, y.device), _f32(C, y.device)
    gamma, beta = torch.ones(C, device=y.device), torch.zeros(C, device=y.device)
    rm, rv, nbt = stats
    ws = _workspace(y.device)
    z = torch.empty_like(y)
    _lib.check(lib.moco_bn_fwd_train(y.data_ptr(), None, z.data_ptr(), N * H * W, C, gamma.data_ptr(), beta.data_ptr(),
                                     rm.data_ptr(), rv.data_ptr(), nbt.data_ptr(), momentum, eps, 1, mean.data_ptr(),
                                     invstd.data_ptr(), ws.data_ptr(), ws.numel(), _lib.cur_stream()), "bn")
    return mean, invstd


def _running(C, dev, g):
    return (torch.rand(C, device=dev, generator=g) - 0.5, torch.rand(C, device=dev, generator=g) + 0.5,
            torch.tensor(7, dtype=torch.long, device=dev))


def _clone(stats):
    return tuple(t.clone() for t in stats)


@pytest.mark.parametrize("side,Cin,Cout", SHAPES)
def test_exact_arithmetic(side, Cin, Cout):
    """x in {-1, 0, 1}, two +-1 entries per weight row: every y is an integer in [-2, 2] and every partial sum is exact.
    y is bit-identical to F.conv2d and to the exact product; the statistics, running statistics and
    num_batches_tracked to what moco_bn_fwd_train computes from that y.  Channel 5 is constant (zero weights)."""
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(side * Cin + Cout)
    N = SMALL_N[side]
    x = _cl(torch.randint(-1, 2, (N, Cin, side, side), device=dev, generator=g).float())
    w = torch.zeros(Cout, Cin, device=dev)
    cols = torch.stack([torch.randperm(Cin, device=dev, generator=g)[:2] for _ in range(Cout)])
    w.scatter_(1, cols, (torch.randint(0, 2, (Cout, 2), device=dev, generator=g) * 2 - 1).float())
    w[5] = 0
    w = w.to(torch.bfloat16).view(Cout, Cin, 1, 1)
    run = _running(Cout, dev, g)
    ours = _clone(run)
    y, mean, invstd = _run(x, w, ours)
    exact = torch.einsum("nchw,oc->nohw", x.double(), w.view(Cout, Cin).double())
    assert torch.equal(y, F.conv2d(x, w))
    assert torch.equal(y, exact.to(torch.bfloat16).contiguous(memory_format=torch.channels_last))
    ref = _clone(run)
    rmean, rinvstd = _bn_stats_of(y, ref)
    torch.cuda.synchronize()
    assert torch.equal(mean, rmean) and torch.equal(invstd, rinvstd)
    for a, b in zip(ours, ref):
        assert torch.equal(a, b)
    assert int(ours[2]) == 8
    eps32 = float(torch.tensor(1e-5, dtype=torch.float32))               # eps reaches the kernel as fp32
    assert float(invstd[5]) == float(torch.tensor(1.0 / math.sqrt(eps32), dtype=torch.float32))


@pytest.mark.parametrize("side,Cin,Cout", SHAPES)
def test_random_full_batch(side, Cin, Cout):
    """Seeded random inputs at batch 256.  y within 1 bf16 ulp of the float64 product, plus the fp32 accumulation
    bound Cin 2^-24 sum |x| |w| that any fp32-accumulating GEMM has where the sum cancels.  mean, invstd, the running
    statistics and num_batches_tracked bit-identical to moco_bn_fwd_train's from that y (the epilogue adds the same
    values in the same order as its statistics pass).  Two calls are bit-identical."""
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(side + Cin * 7 + Cout)
    N = 256
    x = _cl(torch.randn((N, Cin, side, side), device=dev, generator=g) + 0.3)
    w = (torch.randn((Cout, Cin, 1, 1), device=dev, generator=g) * Cin ** -0.5).to(torch.bfloat16)
    run = _running(Cout, dev, g)
    ours = _clone(run)
    y, mean, invstd = _run(x, w, ours)
    M = N * side * side
    xr = x.view(N, Cin, -1).double().transpose(1, 2).reshape(M, Cin)
    ref = xr @ w.view(Cout, Cin).double().t()
    yv = y.permute(0, 2, 3, 1).reshape(M, Cout).double()
    ulp = torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -126))) - 7)
    tol = ulp + Cin * 2.0 ** -24 * (xr.abs() @ w.view(Cout, Cin).double().abs().t())
    assert bool(((yv - ref).abs() <= tol).all()), float(((yv - ref).abs() / tol).max())
    ref_stats = _clone(run)
    rmean, rinvstd = _bn_stats_of(y, ref_stats)
    torch.cuda.synchronize()
    assert torch.equal(mean, rmean) and torch.equal(invstd, rinvstd)
    for a, b in zip(ours, ref_stats):
        assert torch.equal(a, b)
    y2, mean2, invstd2 = _run(x, w, None)
    assert torch.equal(y, y2) and torch.equal(mean, mean2) and torch.equal(invstd, invstd2)


def test_autograd_equals_conv2d_under_autocast(monkeypatch):
    """x.grad and the fp32 weight's gradient through bn.conv1x1_stats equal F.conv2d's under autocast."""
    from moco_b200 import bn
    monkeypatch.setattr(bn, "_conv1x1_wins", lambda M, Cin, Cout: True)
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(11)
    conv = torch.nn.Conv2d(256, 128, 1, bias=False).to(dev).to(memory_format=torch.channels_last)
    norm = bn.BatchNormAct2d(128, relu=True).to(dev)
    x0 = _cl(torch.randn((64, 256, 14, 14), device=dev, generator=g))
    dy = _cl(torch.randn((64, 128, 14, 14), device=dev, generator=g))
    grads = []
    for fused in (True, False):
        x = x0.clone().requires_grad_(True)
        conv.weight.grad = None
        with torch.autocast("cuda", dtype=torch.bfloat16):
            if fused:
                y, st = bn.conv1x1_stats(conv, norm, x)
                assert st is not None and isinstance(y.grad_fn, bn._Conv1x1StatsFn._backward_cls)
            else:
                y = conv(x)
        y.backward(dy)
        grads.append((x.grad, conv.weight.grad))
    assert grads[0][1].dtype == torch.float32
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])


@pytest.mark.parametrize("sc_given", [False, True])
def test_bn_fwd_train_given_equals_the_statistics_passes(sc_given):
    """moco_bn_fwd_train_given with the statistics moco_bn_add_relu_fwd_train computed: the same y and mask bits,
    with one launch (two when the shortcut's statistics are not given), and no running statistics touched."""
    from moco_b200 import _lib
    from moco_b200.bn import _layer, _workspace
    lib = _lib.load()
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(3 + sc_given)
    N, C, H, W = 4, 256, 14, 14
    M = N * H * W
    x, r = _cl(torch.randn((N, C, H, W), device=dev, generator=g)), _cl(torch.randn((N, C, H, W), device=dev, generator=g))
    gam, bet = torch.rand(C, device=dev, generator=g) + 0.5, torch.randn(C, device=dev, generator=g)
    ws = _workspace(dev)
    s = _lib.cur_stream()
    m, i, sm, si = _f32(C, dev), _f32(C, dev), _f32(C, dev), _f32(C, dev)
    run = _running(C, dev, g)
    y1, k1 = torch.empty_like(x), torch.empty((M, C // 8), dtype=torch.uint8, device=dev)
    _lib.check(lib.moco_bn_add_relu_fwd_train(x.data_ptr(), r.data_ptr(), y1.data_ptr(), k1.data_ptr(), M, C,
                                              _layer(gam, bet, m, i, (None, None, None, 0.1, 1e-5)),
                                              _layer(bet.abs(), gam, sm, si, (None, None, None, 0.1, 1e-5)),
                                              ws.data_ptr(), ws.numel(), s), "add_relu")
    y2, k2 = torch.empty_like(x), torch.empty_like(k1)
    rs = _clone(run)
    sm2, si2 = (sm, si) if sc_given else (_f32(C, dev), _f32(C, dev))
    flags = _lib.BN_STATS_GIVEN | (_lib.BN_SC_STATS_GIVEN if sc_given else 0)
    before = _lib.launches
    _lib.check(lib.moco_bn_fwd_train_given(x.data_ptr(), r.data_ptr(), y2.data_ptr(), k2.data_ptr(), M, C, 1,
                                           _layer(gam, bet, m, i, rs + (0.1, 1e-5)),
                                           _layer(bet.abs(), gam, sm2, si2, (None, None, None, 0.1, 1e-5)), flags,
                                           ws.data_ptr(), ws.numel(), s), "given")
    assert _lib.launches == before + (1 if sc_given else 2)
    torch.cuda.synchronize()
    assert torch.equal(y1, y2) and torch.equal(k1, k2)
    for a, b in zip(rs, run):
        assert torch.equal(a, b)


class _CountConvolutions(TorchDispatchMode):
    def __init__(self):
        super().__init__()
        self.n = 0

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        if func is torch.ops.aten.convolution.default:
            self.n += 1
        return func(*args, **(kwargs or {}))


def _conv_ops(fn):
    """(aten.convolution calls, moco_conv1x1_bn_stats calls) of fn()."""
    from moco_b200 import _lib
    lib = _lib.load()
    calls = [0]
    real = lib.moco_conv1x1_bn_stats

    def counted(*args):
        calls[0] += 1
        return real(*args)

    lib.moco_conv1x1_bn_stats = counted
    try:
        with _CountConvolutions() as mode:
            fn()
        torch.cuda.synchronize()
    finally:
        lib.moco_conv1x1_bn_stats = real
    return mode.n, calls[0]


def test_encoder_resnet50_against_cudnn_and_statistics_passes(monkeypatch):
    """ResNet-50 under bf16 autocast with every stride-1 1x1 convolution on moco_conv1x1_bn_stats (the measured-shape
    rule lifted) against the same model on the old dispatch, both measured against the fp32 model: features, the
    gradients of the fc and stem weights and the last running mean are no further from fp32 than the old dispatch's
    (bf16 noise: within 2x, or 5 %); the same total of this library's launches (+1 per rerouted convolution, -1 per
    statistics pass); one aten::convolution fewer per rerouted convolution."""
    from moco_b200 import _lib, bn, encoders
    dev = torch.device("cuda:0")
    torch.manual_seed(5)
    models = [encoders.resnet50(128).to(dev).to(memory_format=torch.channels_last) for _ in range(3)]
    for m in models[1:]:
        m.load_state_dict(models[0].state_dict())
    x = torch.randn(16, 3, 128, 128, device=dev).contiguous(memory_format=torch.channels_last)
    wv = torch.linspace(-1, 1, 128, device=dev)
    rerouted = sum(2 + (blk.short is not None and blk.short[0].stride == (1, 1)) for blk in models[0].layers)
    out = {}

    def step(m, key, autocast=True):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            q = m(x)
        (q * wv).sum().backward()
        out[key] = (q.detach().float(), m.fc.weight.grad.float(), m.stem[0].weight.grad.float(),
                    m.layers[-1].bn3.running_mean.clone())

    step(models[2], "fp32", autocast=False)
    monkeypatch.setattr(bn, "_conv1x1_wins", lambda M, Cin, Cout: True)
    before = _lib.launches
    ops_a, kern_a = _conv_ops(lambda: step(models[0], "new"))
    launches_a = _lib.launches - before
    monkeypatch.setattr(bn, "_conv1x1_ok", lambda *args: False)
    before = _lib.launches
    ops_b, kern_b = _conv_ops(lambda: step(models[1], "old"))
    launches_b = _lib.launches - before
    assert kern_a == rerouted and kern_b == 0
    assert ops_b - ops_a == rerouted, (ops_a, ops_b, rerouted)
    assert launches_a == launches_b
    for i, name in enumerate(("q", "fc.weight.grad", "stem weight.grad", "last running_mean")):
        ref = out["fp32"][i]
        e_new = float((out["new"][i] - ref).norm() / ref.norm())
        e_old = float((out["old"][i] - ref).norm() / ref.norm())
        assert e_new < max(2.0 * e_old, 0.05), (name, e_new, e_old)
    assert torch.equal(models[0].layers[0].bn1.num_batches_tracked, models[1].layers[0].bn1.num_batches_tracked)


def test_resnet18_keeps_the_old_path():
    """_Basic blocks keep cuDNN's convolutions (their only 1x1 convolutions are stride 2): no conv1x1 kernel, and the
    same launches as with the conv1x1 path switched off."""
    from moco_b200 import _lib, encoders
    dev = torch.device("cuda:0")
    torch.manual_seed(2)
    m = encoders.resnet18(128).to(dev).to(memory_format=torch.channels_last)
    x = torch.randn(64, 3, 224, 224, device=dev).contiguous(memory_format=torch.channels_last)
    before = _lib.launches

    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            q = m(x)
        q.float().sum().backward()

    ops, kern = _conv_ops(step)
    assert kern == 0
    n_fwd_bwd = _lib.launches - before
    from moco_b200 import bn
    bn_ok = bn._conv1x1_ok
    try:
        bn._conv1x1_ok = lambda *args: False
        before = _lib.launches
        _conv_ops(step)
        assert _lib.launches - before == n_fwd_bwd
    finally:
        bn._conv1x1_ok = bn_ok
