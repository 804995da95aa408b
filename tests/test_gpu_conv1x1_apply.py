"""moco_conv1x1_bn_add_relu_fwd (csrc/conv1x1_sm90.cu) against moco_conv1x1_bn_stats + moco_bn_fwd_train_given on the
same inputs, and its wiring in ResNet-50 (bn.conv1x1_bn_add_relu) against the same model on the unfused path."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# (Cin, Cout, N, H, W): conv3 of every table shape at batch 256, a ragged M, a small M, and BN = 64 (Cout = 64)
SHAPES = [(64, 256, 256, 56, 56), (128, 512, 256, 28, 28), (256, 1024, 256, 14, 14),
          (64, 256, 3, 13, 13), (128, 512, 1, 8, 16), (64, 64, 2, 9, 7)]


def _cl(t):
    return t.bfloat16().contiguous(memory_format=torch.channels_last)


class _Bn:
    """One BatchNorm's tensors (fresh running statistics) and its moco_bn_layer."""

    def __init__(self, C, g, dev):
        self.gamma = torch.rand(C, device=dev, generator=g) + 0.5
        self.beta = torch.randn(C, device=dev, generator=g)
        self.rm, self.rv = torch.zeros(C, device=dev), torch.ones(C, device=dev)
        self.nbt = torch.zeros((), dtype=torch.long, device=dev)
        self.mean, self.invstd = torch.empty(C, device=dev), torch.empty(C, device=dev)

    def copy(self):
        other = object.__new__(_Bn)
        for k, v in vars(self).items():
            setattr(other, k, v.clone())
        return other

    def layer(self):
        from moco_b200.bn import _layer
        return _layer(self.gamma, self.beta, self.mean, self.invstd, (self.rm, self.rv, self.nbt, 0.1, 1e-5))

    def state(self):
        return [self.mean, self.invstd, self.rm, self.rv, self.nbt]


def _inputs(Cin, C, N, H, W, exact, seed):
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(seed)
    if exact:     # h = a . w is exact in any summation order: halves times {-1, 0, 1}
        a = _cl(torch.randint(-2, 3, (N, Cin, H, W), device=dev, generator=g) * 0.5)
        w = torch.randint(-1, 2, (C, Cin, 1, 1), device=dev, generator=g).bfloat16()
    else:
        a = _cl(torch.randn((N, Cin, H, W), device=dev, generator=g))
        w = (torch.randn((C, Cin, 1, 1), device=dev, generator=g) * Cin ** -0.5).bfloat16()
    r = _cl(torch.randn((N, C, H, W), device=dev, generator=g) * 2)
    return a, w, r, _Bn(C, g, dev), _Bn(C, g, dev)


def _ws(lib, dev):
    return torch.zeros(max(lib.moco_conv1x1_workspace_bytes(), lib.moco_bn_workspace_bytes()), dtype=torch.uint8,
                       device=dev)


def _unfused(a, w, r, bn, sc):
    from moco_b200 import _lib
    lib = _lib.load()
    N, Cin, H, W = a.shape
    C, M = w.shape[0], N * H * W
    ws = _ws(lib, a.device)
    h = torch.empty((N, C, H, W), dtype=torch.bfloat16, device=a.device, memory_format=torch.channels_last)
    y, mask = torch.empty_like(h), torch.empty((M, C // 8), dtype=torch.uint8, device=a.device)
    _lib.check(lib.moco_conv1x1_bn_stats(a.data_ptr(), w.data_ptr(), h.data_ptr(), M, Cin, C, bn.layer(),
                                         ws.data_ptr(), ws.numel(), _lib.cur_stream()), "moco_conv1x1_bn_stats")
    _lib.check(lib.moco_bn_fwd_train_given(h.data_ptr(), r.data_ptr(), y.data_ptr(), mask.data_ptr(), M, C, 1,
                                           bn.layer(), sc.layer() if sc else None, _lib.BN_STATS_GIVEN, ws.data_ptr(),
                                           ws.numel(), _lib.cur_stream()), "moco_bn_fwd_train_given")
    torch.cuda.synchronize()
    return y, mask


def _fused(a, w, r, bn, sc, given):
    from moco_b200 import _lib
    lib = _lib.load()
    N, Cin, H, W = a.shape
    C, M = w.shape[0], N * H * W
    ws = _ws(lib, a.device)
    y = torch.empty((N, C, H, W), dtype=torch.bfloat16, device=a.device, memory_format=torch.channels_last)
    mask = torch.empty((M, C // 8), dtype=torch.uint8, device=a.device)
    if given:
        h = torch.empty_like(y)
        _lib.check(lib.moco_conv1x1_bn_stats(a.data_ptr(), w.data_ptr(), h.data_ptr(), M, Cin, C, bn.layer(),
                                             ws.data_ptr(), ws.numel(), _lib.cur_stream()), "moco_conv1x1_bn_stats")
    before = _lib.launches
    _lib.check(lib.moco_conv1x1_bn_add_relu_fwd(a.data_ptr(), w.data_ptr(), r.data_ptr(), y.data_ptr(),
                                                mask.data_ptr(), M, Cin, C, bn.layer(), sc.layer() if sc else None,
                                                _lib.BN_STATS_GIVEN if given else 0, ws.data_ptr(), ws.numel(),
                                                _lib.cur_stream()), "moco_conv1x1_bn_add_relu_fwd")
    assert _lib.launches == before + 1 + (not given) + (sc is not None)
    torch.cuda.synchronize()
    return y, mask


def _check(Cin, C, N, H, W, shortcut, given, exact, seed):
    a, w, r, bn, sc = _inputs(Cin, C, N, H, W, exact, seed)
    sc = sc if shortcut else None
    bn2, sc2 = bn.copy(), sc.copy() if sc else None
    y0, m0 = _unfused(a, w, r, bn, sc)
    y1, m1 = _fused(a, w, r, bn2, sc2, given)
    assert torch.equal(y0, y1)
    assert torch.equal(m0, m1)
    assert float((y0 > 0).float().mean()) > 0.2                   # the ReLU and the mask bits are exercised
    for u, v in zip(bn.state() + (sc.state() if sc else []), bn2.state() + (sc2.state() if sc2 else [])):
        assert torch.equal(u, v)
    return a, w, r, bn, sc, y1, m1


@pytest.mark.parametrize("given", [True, False])
@pytest.mark.parametrize("shortcut", [False, True])
@pytest.mark.parametrize("shape", SHAPES)
def test_matches_unfused_exact(shape, shortcut, given):
    """Exact-arithmetic inputs: y, the mask bits, the statistics and the running statistics (the shortcut BN's too)
    bit-identical to the unfused calls, with the statistics given and computed in the call."""
    _check(*shape, shortcut, given, True, sum(shape))


@pytest.mark.parametrize("shortcut", [False, True])
@pytest.mark.parametrize("shape", SHAPES[:3])
def test_matches_unfused_seeded(shape, shortcut):
    """Seeded random inputs at batch 256: the recomputed tile is the h the statistics pass stores, so y is still
    bit-identical, and a second call is bit-identical to the first."""
    a, w, r, bn, sc, y1, m1 = _check(*shape, shortcut, False, False, 7 + sum(shape))
    y2, m2 = _fused(a, w, r, bn.copy(), sc.copy() if sc else None, False)
    assert torch.equal(y1, y2) and torch.equal(m1, m2)


def test_resnet50_query_and_key_bit_identical(monkeypatch):
    """ResNet-50 at 16 x 224^2 under bf16 autocast, every conv3 of the table on the new path (the M bound of the table
    lifted) against the same model with the table emptied: a training step (query) gives bit-identical features,
    parameter gradients and running buffers with the same launch total, and so does a forward without grad (key),
    which never asks for conv3's output."""
    from moco_b200 import _lib, bn, encoders
    dev = torch.device("cuda:0")
    torch.manual_seed(5)
    models = [encoders.resnet50(128).to(dev).to(memory_format=torch.channels_last) for _ in range(2)]
    models[1].load_state_dict(models[0].state_dict())
    x = torch.randn(16, 3, 224, 224, device=dev).contiguous(memory_format=torch.channels_last)
    wv = torch.linspace(-1, 1, 128, device=dev)
    lib = _lib.load()
    real = lib.moco_conv1x1_bn_add_relu_fwd
    flags = []

    def spy(*args):
        flags.append(args[10])
        return real(*args)

    monkeypatch.setattr(lib, "moco_conv1x1_bn_add_relu_fwd", spy)
    monkeypatch.setattr(bn, "_conv1x1_wins", lambda M, Cin, Cout: True)       # both arms: conv1x1_stats everywhere
    wins = lambda M, Cin, Cout, key, sc: (Cin, Cout, key, sc) in bn._APPLY_WINS
    sites = {key: sum(1 for b in models[0].layers if wins(0, *b.conv3.weight.shape[1::-1], key, b.short is not None))
             for key in (False, True)}
    assert sites[True] == 13

    def run(m, new, grad):
        monkeypatch.setattr(bn, "_apply_wins", wins if new else (lambda *a: False))
        del flags[:]
        before = _lib.launches
        with torch.set_grad_enabled(grad), torch.autocast("cuda", dtype=torch.bfloat16):
            q = m(x)
        if grad:
            (q * wv).sum().backward()
        torch.cuda.synchronize()
        grads = [p.grad.clone() for p in m.parameters()] if grad else []
        return q.float(), grads, [t.clone() for t in m.buffers()], _lib.launches - before, list(flags)

    for grad in (True, False):
        q1, g1, b1, n1, f1 = run(models[0], True, grad)
        q0, g0, b0, n0, f0 = run(models[1], False, grad)
        assert f0 == [] and len(f1) == sites[not grad]
        assert all((f & _lib.BN_STATS_GIVEN) == (_lib.BN_STATS_GIVEN if grad else 0) for f in f1)
        assert n1 == n0
        assert torch.equal(q1, q0)
        for u, v in zip(g1 + b1, g0 + b0):
            assert torch.equal(u, v)
