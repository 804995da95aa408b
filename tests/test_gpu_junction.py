"""A block input's two gradients summed inside its producer's backward (moco_bn_add_relu_bwd2, moco_maxpool3x3s2_bwd2
and the hand-over of bn.py) against autograd's separate bf16 add followed by the one-gradient entry points: every
gradient, parameter gradient and buffer bit-identical.  Also the max pool's tie and NaN rules at the pool kernels'
tiling, against an exact torch emulation of torch's rule."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SHAPES = [(5, 64, 9, 9), (3, 256, 7, 7), (2, 2048, 7, 5), (4, 256, 14, 14)]
POOL_SHAPES = [(4, 64, 112, 112), (3, 64, 9, 11), (2, 256, 7, 6), (5, 64, 1, 3), (2, 64, 2, 2), (3, 16, 10, 7)]


def _cl(t):
    return t.bfloat16().contiguous(memory_format=torch.channels_last)


def _bn(C, dev, g, relu):
    from moco_b200.bn import BatchNormAct2d
    mod = BatchNormAct2d(C, relu=relu).to(dev)
    with torch.no_grad():
        mod.weight.copy_(torch.rand(C, device=dev, generator=g) + 0.5)
        mod.bias.copy_(torch.randn(C, device=dev, generator=g) * 0.3)
    return mod


def _f32(C, dev):
    return torch.empty(C, dtype=torch.float32, device=dev)


@pytest.mark.parametrize("shortcut", [False, True])
@pytest.mark.parametrize("N,C,H,W", SHAPES)
def test_bn_add_relu_bwd2_equals_the_add_then_bwd(N, C, H, W, shortcut):
    from moco_b200 import _lib
    from moco_b200.bn import _layer
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(N * C + H + shortcut)
    lib = _lib.load()
    M = N * H * W
    x, r = _cl(torch.randn((N, C, H, W), device=dev, generator=g)), _cl(torch.randn((N, C, H, W), device=dev, generator=g))
    dy, dy2 = _cl(torch.randn((N, C, H, W), device=dev, generator=g)), _cl(torch.randn((N, C, H, W), device=dev, generator=g))
    dy2[:, 3] = -dy[:, 3]                                      # exact cancellations
    w, b = torch.rand(C, device=dev, generator=g) + 0.5, torch.randn(C, device=dev, generator=g)
    ws = torch.zeros(lib.moco_bn_workspace_bytes(), dtype=torch.uint8, device=dev)
    s = _lib.cur_stream()
    mean, invstd, sm, si = _f32(C, dev), _f32(C, dev), _f32(C, dev), _f32(C, dev)
    y = torch.empty_like(x)
    mask = torch.empty((M, C // 8), dtype=torch.uint8, device=dev)
    sc = _layer(w, b, sm, si, (None, None, None, 0.1, 1e-5)) if shortcut else None
    assert lib.moco_bn_add_relu_fwd_train(x.data_ptr(), r.data_ptr(), y.data_ptr(), mask.data_ptr(), M, C,
                                          _layer(w, b, mean, invstd, (None, None, None, 0.1, 1e-5)), sc,
                                          ws.data_ptr(), ws.numel(), s) == 0

    def run(two):
        dx, dres = torch.empty_like(x), torch.empty_like(x)
        dg, db, sdg, sdb = _f32(C, dev), _f32(C, dev), _f32(C, dev), _f32(C, dev)
        bn = _layer(w, None, mean, invstd, dgamma=dg, dbeta=db)
        scl = _layer(w, None, sm, si, dgamma=sdg, dbeta=sdb) if shortcut else None
        res = r.data_ptr() if shortcut else None
        before = _lib.launches
        if two:
            rc = lib.moco_bn_add_relu_bwd2(dy.data_ptr(), dy2.data_ptr(), x.data_ptr(), res, mask.data_ptr(), M, C, bn,
                                           scl, dx.data_ptr(), dres.data_ptr(), ws.data_ptr(), ws.numel(), s)
        else:
            tot = dy + dy2                                     # autograd's bf16 add
            rc = lib.moco_bn_add_relu_bwd(tot.data_ptr(), x.data_ptr(), res, mask.data_ptr(), M, C, bn, scl,
                                          dx.data_ptr(), dres.data_ptr(), ws.data_ptr(), ws.numel(), s)
        assert rc == 0 and _lib.launches == before + 2
        torch.cuda.synchronize()
        return dx, dres, dg, db, sdg, sdb

    a, b2 = run(True), run(False)
    for name, u, v in zip(("dx", "dres", "dgamma", "dbeta", "sc_dgamma", "sc_dbeta"), a, b2):
        if name.startswith("sc_") and not shortcut:
            continue
        assert torch.equal(u, v), name


def _pool_reference(x):
    """y, tap bytes and the tap rule of torch's max_pool2d (3x3 / 2 / pad 1): taps scanned kh then kw, the first
    in-image tap starts the window, later ones replace on `v > max || isnan(v)`."""
    N, C, H, W = x.shape
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    xp = F.pad(x.float(), (1, 2, 1, 2))
    valid = F.pad(torch.ones((N, C, H, W), device=x.device), (1, 2, 1, 2)) > 0
    m = torch.full((N, C, OH, OW), float("-inf"), device=x.device)
    tap = torch.zeros((N, C, OH, OW), dtype=torch.uint8, device=x.device)
    first = torch.ones((N, C, OH, OW), dtype=torch.bool, device=x.device)
    for kh in range(3):
        for kw in range(3):
            v = xp[:, :, kh:kh + 2 * OH:2, kw:kw + 2 * OW:2]
            ok = valid[:, :, kh:kh + 2 * OH:2, kw:kw + 2 * OW:2]
            upd = ok & (first | (v > m) | torch.isnan(v))
            m = torch.where(upd, v, m)
            tap = torch.where(upd, torch.full_like(tap, kh * 3 + kw), tap)
            first = first & ~ok
    return m, tap


def _pool_bwd_reference(g, tap, H, W):
    """dx of the gather: each pixel adds its windows' gradients in increasing (oh, ow) order in fp32 (taps kh, kw
    decreasing), one rounding to bf16."""
    N, C, OH, OW = g.shape
    dxp = torch.zeros((N, C, 2 * OH + 2, 2 * OW + 2), device=g.device)
    for kh in (2, 1, 0):
        for kw in (2, 1, 0):
            sl = dxp[:, :, kh:kh + 2 * OH:2, kw:kw + 2 * OW:2]
            sl += torch.where(tap == kh * 3 + kw, g.float(), torch.zeros_like(sl))
    return dxp[:, :, 1:H + 1, 1:W + 1].bfloat16()


@pytest.mark.parametrize("N,C,H,W", POOL_SHAPES)
def test_maxpool_ties_nan_and_bwd2_at_the_kernel_tiling(N, C, H, W):
    from moco_b200 import _lib
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(N * 31 + H * 7 + W)
    lib = _lib.load()
    s = _lib.cur_stream()
    # few distinct values (ties everywhere), some NaN (also several in one window), some -inf
    x = torch.randint(-2, 3, (N, C, H, W), device=dev, generator=g).float()
    x[torch.rand((N, C, H, W), device=dev, generator=g) < 0.03] = float("nan")
    x[torch.rand((N, C, H, W), device=dev, generator=g) < 0.02] = float("-inf")
    x = _cl(x)
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    y = torch.empty((N, C, OH, OW), dtype=torch.bfloat16, device=dev, memory_format=torch.channels_last)
    taps = torch.empty((N, OH, OW, C), dtype=torch.uint8, device=dev)
    assert lib.moco_maxpool3x3s2_fwd(x.data_ptr(), y.data_ptr(), taps.data_ptr(), N, H, W, C, s) == 0
    m, tap = _pool_reference(x)
    torch.cuda.synchronize()
    assert torch.equal(taps, tap.permute(0, 2, 3, 1))
    assert torch.equal(torch.isnan(y), torch.isnan(m)) and torch.equal(y[~torch.isnan(y)], m.bfloat16()[~torch.isnan(m)])
    assert bool(torch.isnan(y).any()) or H * W < 16
    dy = _cl(torch.randn((N, C, OH, OW), device=dev, generator=g))
    dy2 = _cl(torch.randn((N, C, OH, OW), device=dev, generator=g))
    dy2[:, 0] = -dy[:, 0]
    dx1, dx2 = torch.empty_like(x), torch.empty_like(x)
    before = _lib.launches
    assert lib.moco_maxpool3x3s2_bwd(dy.data_ptr(), taps.data_ptr(), dx1.data_ptr(), N, H, W, C, s) == 0
    assert lib.moco_maxpool3x3s2_bwd2(dy.data_ptr(), dy2.data_ptr(), taps.data_ptr(), dx2.data_ptr(), N, H, W, C,
                                      s) == 0
    assert _lib.launches == before + 2
    tot = dy + dy2                                             # autograd's bf16 add
    dx3 = torch.empty_like(x)
    assert lib.moco_maxpool3x3s2_bwd(tot.data_ptr(), taps.data_ptr(), dx3.data_ptr(), N, H, W, C, s) == 0
    torch.cuda.synchronize()
    assert torch.equal(dx1, _pool_bwd_reference(dy, tap, H, W))
    assert torch.equal(dx3, _pool_bwd_reference(tot, tap, H, W))
    assert torch.equal(dx2, dx3)


def _two_consumers(y, d1, d2, hand):
    """A block input's two consumers: the first convolution's branch and, through the hand-over, the residual's."""
    from moco_b200 import bn
    r = bn.hand_over(y) if hand else y
    return (y.float() * d1.float()).sum() + (r.float() * d2.float()).sum()


@pytest.mark.parametrize("shortcut", [False, True])
@pytest.mark.parametrize("N,C,H,W", SHAPES[:2])
def test_handed_gradient_in_the_block_producer(N, C, H, W, shortcut):
    from moco_b200 import _lib, bn
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(N + C + shortcut)
    x, r = _cl(torch.randn((N, C, H, W), device=dev, generator=g)), _cl(torch.randn((N, C, H, W), device=dev, generator=g))
    d1, d2 = _cl(torch.randn((N, C, H, W), device=dev, generator=g)), _cl(torch.randn((N, C, H, W), device=dev, generator=g))
    out = {}
    for hand in (True, False):
        torch.manual_seed(0)
        mod = _bn(C, dev, torch.Generator(device=dev).manual_seed(5), True)
        sc = _bn(C, dev, torch.Generator(device=dev).manual_seed(6), False) if shortcut else None
        xa, ra = x.clone().requires_grad_(True), r.clone().requires_grad_(True)
        y = mod(xa, ra, shortcut_bn=sc)
        assert isinstance(y.grad_fn, bn._BatchNormAddReluFn._backward_cls)
        loss = _two_consumers(y, d1, d2, hand)
        before = _lib.launches
        loss.backward(retain_graph=True)
        assert _lib.launches == before + 2
        first = [t.grad.clone() for t in (xa, ra, mod.weight, mod.bias)]
        for t in (xa, ra, mod.weight, mod.bias):
            t.grad = None
        loss.backward()                                        # the handed gradient is taken once per backward
        assert all(torch.equal(a, t.grad) for a, t in zip(first, (xa, ra, mod.weight, mod.bias)))
        out[hand] = first
    for name, a, b in zip(("dx", "dresidual", "dgamma", "dbeta"), out[True], out[False]):
        assert torch.equal(a, b), name


@pytest.mark.parametrize("N,C,H,W", [(4, 64, 112, 112), (3, 64, 9, 11)])
def test_handed_gradient_in_the_stem_producer(N, C, H, W):
    from moco_b200 import _lib, bn
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(H + W)
    x = _cl(torch.randint(-3, 4, (N, C, H, W), device=dev, generator=g).float() * 0.5)
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    d1, d2 = _cl(torch.randn((N, C, OH, OW), device=dev, generator=g)), _cl(torch.randn((N, C, OH, OW), device=dev, generator=g))
    out = {}
    for hand in (True, False):
        mod = _bn(C, dev, torch.Generator(device=dev).manual_seed(5), True)
        xa = x.clone().requires_grad_(True)
        y = mod.forward_maxpool(xa, bn.MaxPool3x3s2())
        assert isinstance(y.grad_fn, bn._BatchNormReluMaxPoolFn._backward_cls)
        before = _lib.launches
        _two_consumers(y, d1, d2, hand).backward()
        assert _lib.launches == before + 3                     # pool backward + the BatchNorm's two passes
        out[hand] = (xa.grad, mod.weight.grad, mod.bias.grad)
    for name, a, b in zip(("dx", "dgamma", "dbeta"), out[True], out[False]):
        assert torch.equal(a, b), name


def test_hand_over_only_for_its_own_producers():
    from moco_b200 import bn
    dev = torch.device("cuda:0")
    x0 = _cl(torch.randn((2, 64, 5, 5), device=dev)).requires_grad_(True)
    x = x0 * 2                                                 # a producer that is not one of ours
    assert bn.hand_over(x) is x
    mod = _bn(64, dev, torch.Generator(device=dev).manual_seed(1), True)
    y = mod(x, _cl(torch.randn((2, 64, 5, 5), device=dev)))
    assert bn.hand_over(y) is not y
    with torch.no_grad():
        assert bn.hand_over(y) is y
    bn.set_fused(False)
    try:
        assert bn.hand_over(y) is y
    finally:
        bn.set_fused(True)


def _bf16_adds(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if "CUDAFunctor_add<c10::BFloat16>" in e.name and e.device_time > 0)


@pytest.mark.parametrize("arch", ["resnet50", "resnet18"])
def test_encoder_hand_over_equals_the_autograd_sum(arch, monkeypatch):
    """Whole encoder under bf16 autocast: with the hand-over against the same fused model whose block inputs are
    summed by autograd -- outputs, parameter gradients and buffers bit-identical, no bf16 add left in the backward,
    the same number of this library's launches, and a retained graph's second backward gives the same gradients."""
    from moco_b200 import _lib, bn, encoders
    dev = torch.device("cuda:0")
    torch.manual_seed(3)
    ctor = getattr(encoders, arch)
    a = ctor(128).to(dev).to(memory_format=torch.channels_last)
    b = ctor(128).to(dev).to(memory_format=torch.channels_last)
    b.load_state_dict(a.state_dict())
    x = torch.randn(8, 3, 96, 96, device=dev).contiguous(memory_format=torch.channels_last)
    w = torch.linspace(-1, 1, 128, device=dev)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        qa = a(x)
    la = (qa * w).sum()
    before = _lib.launches
    adds_a = _bf16_adds(lambda: la.backward(retain_graph=True))
    launches_a = _lib.launches - before
    grads = [p.grad.clone() for p in a.parameters()]
    a.zero_grad(set_to_none=True)
    la.backward()
    assert all(torch.equal(g0, p.grad) for g0, p in zip(grads, a.parameters()))

    monkeypatch.setattr(bn, "hand_over", lambda t: t)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        qb = b(x)
    assert torch.equal(qa, qb)
    before = _lib.launches
    adds_b = _bf16_adds(lambda: (qb * w).sum().backward())
    assert _lib.launches - before == launches_a
    assert adds_a == 0 and adds_b == len(b.layers), (adds_a, adds_b)
    for (na, pa), (nb, pb) in zip(a.named_parameters(), b.named_parameters()):
        assert torch.equal(pa.grad, pb.grad), na
    for (na, ba), (nb, bb) in zip(a.named_buffers(), b.named_buffers()):
        assert torch.equal(ba, bb), na
