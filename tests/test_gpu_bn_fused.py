"""The residual BatchNorm paths of moco_bn_add_relu_fwd_train / moco_bn_add_relu_bwd (ReLU mask as bits; a downsample
block's shortcut BN folded in) against the unfused sequence on moco_bn_fwd_train / moco_bn_bwd, on the same inputs:
every output, gradient, running statistic and step counter must be bit-identical."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _cl(t):
    return t.bfloat16().contiguous(memory_format=torch.channels_last)


def _bn(C, dev, g, relu):
    from moco_b200.bn import BatchNormAct2d
    mod = BatchNormAct2d(C, relu=relu).to(dev)
    with torch.no_grad():
        mod.weight.copy_(torch.rand(C, device=dev, generator=g) + 0.5)
        mod.bias.copy_(torch.randn(C, device=dev, generator=g) * 0.3)
        mod.running_mean.copy_(torch.randn(C, device=dev, generator=g))
        mod.running_var.copy_(torch.rand(C, device=dev, generator=g) + 0.5)
        # channel 1: gamma so small that positive outputs underflow to zero in bf16 (mask from the rounded value)
        mod.weight[1] = 1e-42
        mod.bias[1] = 0.0
    return mod


def _clone(mod):
    from moco_b200.bn import BatchNormAct2d
    c = BatchNormAct2d(mod.num_features, relu=mod.relu).to(mod.weight.device)
    c.load_state_dict(mod.state_dict())
    return c


def _unfused(mod, x, r):
    from moco_b200.bn import _BatchNormActFn
    return _BatchNormActFn.apply(x, mod.weight, mod.bias, r, mod.running_mean, mod.running_var, mod.num_batches_tracked,
                                 mod.momentum, mod.eps, mod.relu)


def _inputs(shape, dev, g):
    x = _cl(torch.randn(shape, device=dev, generator=g) * 1.5 + 0.4)
    r = torch.randn(shape, device=dev, generator=g)
    r[:, 1] = 0.0                                                 # the underflow channel: y = bf16(tiny) = 0
    r[:, 2] = -1e4                                                # exact ReLU zeros over a whole channel
    return x, _cl(r), _cl(torch.randn(shape, device=dev, generator=g))


def _same_module_state(a, b):
    for n in ("running_mean", "running_var", "num_batches_tracked"):
        assert torch.equal(getattr(a, n), getattr(b, n)), n
    assert torch.equal(a.weight.grad, b.weight.grad) and torch.equal(a.bias.grad, b.bias.grad)


# C in {64, 256, 2048}; M = N * H * W not a multiple of 32
SHAPES = [(5, 64, 9, 9), (3, 256, 7, 7), (2, 2048, 7, 5), (4, 256, 14, 14)]


@pytest.mark.parametrize("N,C,H,W", SHAPES)
def test_mask_bits_path_is_bit_identical(N, C, H, W):
    import moco_b200._lib as L
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(N * C + H)
    mod = _bn(C, dev, g, True)
    ref = _clone(mod)
    x, r, dy = _inputs((N, C, H, W), dev, g)
    xa, ra = x.clone().requires_grad_(True), r.clone().requires_grad_(True)
    xb, rb = x.clone().requires_grad_(True), r.clone().requires_grad_(True)
    before = L.launches
    ya = mod(xa, ra)
    assert L.launches == before + 2
    yb = _unfused(ref, xb, rb)
    assert torch.equal(ya, yb)
    assert bool((ya == 0).any()) and bool((ya > 0).any())
    ya.backward(dy)
    yb.backward(dy)
    assert torch.equal(xa.grad, xb.grad) and torch.equal(ra.grad, rb.grad)
    _same_module_state(mod, ref)
    # no grad (the key encoder): no mask, same output
    with torch.no_grad():
        assert torch.equal(mod(x, r), _unfused(ref, x, r))
    assert torch.equal(mod.running_var, ref.running_var)


@pytest.mark.parametrize("N,C,H,W", SHAPES)
def test_shortcut_bn_folded_in_is_bit_identical(N, C, H, W):
    import moco_b200._lib as L
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(7 + N * C + H)
    bn3, sc = _bn(C, dev, g, True), _bn(C, dev, g, False)
    ref3, refsc = _clone(bn3), _clone(sc)
    x, xds, dy = _inputs((N, C, H, W), dev, g)
    xds = _cl(torch.randn((N, C, H, W), device=dev, generator=g) * 0.7 - 0.2)
    xa, da = x.clone().requires_grad_(True), xds.clone().requires_grad_(True)
    xb, db = x.clone().requires_grad_(True), xds.clone().requires_grad_(True)
    before = L.launches
    ya = bn3(xa, da, shortcut_bn=sc)
    assert L.launches == before + 3
    yb = _unfused(ref3, xb, _unfused(refsc, db, None))
    assert torch.equal(ya, yb)
    before = L.launches
    ya.backward(dy)
    assert L.launches == before + 2
    yb.backward(dy)
    assert torch.equal(xa.grad, xb.grad), "dx"
    assert torch.equal(da.grad, db.grad), "dx_ds"
    _same_module_state(bn3, ref3)
    _same_module_state(sc, refsc)
    with torch.no_grad():
        assert torch.equal(bn3(x, xds, shortcut_bn=sc), _unfused(ref3, x, _unfused(refsc, xds, None)))
    assert int(sc.num_batches_tracked) == int(refsc.num_batches_tracked) == 2


def test_shortcut_bn_falls_back_where_the_kernels_do_not_apply():
    """fp32 activations (and set_fused(False)): the shortcut BN runs as its own module, then the add and the ReLU."""
    from moco_b200 import bn
    import torch.nn.functional as F
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(11)
    bn3, sc = _bn(64, dev, g, True), _bn(64, dev, g, False)
    ref3, refsc = torch.nn.BatchNorm2d(64).to(dev), torch.nn.BatchNorm2d(64).to(dev)
    ref3.load_state_dict(bn3.state_dict())
    refsc.load_state_dict(sc.state_dict())
    x = torch.randn(4, 64, 6, 6, device=dev, generator=g)
    xds = torch.randn(4, 64, 6, 6, device=dev, generator=g)
    assert torch.equal(bn3(x, xds, shortcut_bn=sc), F.relu(ref3(x) + refsc(xds)))
    bn.set_fused(False)
    try:
        xc, dc = _cl(x), _cl(xds)
        assert torch.equal(bn3(xc, dc, shortcut_bn=sc), F.relu(ref3(xc) + refsc(dc)))
    finally:
        bn.set_fused(True)


@pytest.mark.parametrize("arch", ["resnet50", "resnet18"])
def test_encoder_fused_is_as_close_to_fp32_as_the_torch_bf16_ops(arch):
    """Whole encoder forward + backward with every fused path (bounds of test_gpu_bn's ResNet-50 closeness test)."""
    from moco_b200 import encoders, bn
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    ctor = getattr(encoders, arch)
    models = [ctor(128).to(dev).to(memory_format=torch.channels_last) for _ in range(3)]
    for m in models[1:]:
        m.load_state_dict(models[0].state_dict())
    x = torch.randn(16, 3, 224, 224, device=dev).contiguous(memory_format=torch.channels_last)
    w = torch.linspace(-1, 1, 128, device=dev)
    outs = []
    for mod, mode in zip(models, ("fused", "torch_bf16", "fp32")):
        bn.set_fused(mode == "fused")
        try:
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=mode != "fp32"):
                q = mod(x)
            (q * w).sum().backward()
        finally:
            bn.set_fused(True)
        down = next(b for b in mod.layers if b.short is not None and b.short[0].stride != (1, 1))
        outs.append((q.detach().float(), mod.fc.weight.grad.float().clone(), mod.stem[0].weight.grad.float().clone(),
                     down.short[0].weight.grad.float().clone(), mod.stem[1].running_var.clone(),
                     down.short[1].running_mean.clone()))
    fused, torch_bf16, fp32 = outs
    for i, name in enumerate(("q", "fc.weight.grad", "stem conv weight.grad", "shortcut conv weight.grad")):
        e_f = float((fused[i] - fp32[i]).norm() / fp32[i].norm())
        e_t = float((torch_bf16[i] - fp32[i]).norm() / fp32[i].norm())
        assert e_f < max(2.0 * e_t, 0.05), (name, e_f, e_t)
    assert float(((fused[4] - fp32[4]).abs() / fp32[4]).max()) < 2e-2
    e_f = float((fused[5] - fp32[5]).norm() / fp32[5].norm())
    e_t = float((torch_bf16[5] - fp32[5]).norm() / fp32[5].norm())
    assert e_f < max(2.0 * e_t, 0.05), ("shortcut running_mean", e_f, e_t)


# odd and even H / W; C = 64 (the stem) and 256
POOL_SHAPES = [(4, 64, 112, 112), (3, 64, 9, 11), (2, 256, 7, 6), (5, 64, 1, 3)]


@pytest.mark.parametrize("N,C,H,W", POOL_SHAPES)
def test_stem_bn_relu_maxpool_is_bit_identical(N, C, H, W):
    """BatchNorm + ReLU folded into the 3x3/2 max pool against moco_bn_fwd_train + moco_maxpool3x3s2_fwd and
    moco_maxpool3x3s2_bwd + moco_bn_bwd: pooled y, tap bytes, dx, dgamma, dbeta, running statistics."""
    from moco_b200 import _lib
    from moco_b200.bn import MaxPool3x3s2, _MaxPool3x3s2Fn, _layer
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(N * 100 + H * 7 + W)
    mod = _bn(C, dev, g, True)
    ref = _clone(mod)
    # few distinct values: many pool ties besides the ReLU zeros; channel 1 underflows to zero in bf16
    x = _cl(torch.randint(-3, 4, (N, C, H, W), device=dev, generator=g).float() * 0.5)
    dy = _cl(torch.randn((N, C, (H - 1) // 2 + 1, (W - 1) // 2 + 1), device=dev, generator=g))
    xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    before = _lib.launches
    ya = mod.forward_maxpool(xa, MaxPool3x3s2())
    assert _lib.launches == before + 2
    yb = _MaxPool3x3s2Fn.apply(_unfused(ref, xb, None))
    assert torch.equal(ya, yb)
    ya.backward(dy)
    yb.backward(dy)
    assert torch.equal(xa.grad, xb.grad), "dx"
    _same_module_state(mod, ref)
    # the tap bytes, through the C entry points
    lib = _lib.load()
    ws = torch.zeros(lib.moco_bn_workspace_bytes(), dtype=torch.uint8, device=dev)
    y1, y2 = torch.empty_like(ya), torch.empty_like(ya)
    t1 = torch.empty((N, ya.shape[2], ya.shape[3], C), dtype=torch.uint8, device=dev)
    t2 = torch.empty_like(t1)
    f32 = lambda: torch.empty(C, dtype=torch.float32, device=dev)
    m1, i1, m2, i2 = f32(), f32(), f32(), f32()
    s = _lib.cur_stream()
    w, b = mod.weight.detach(), mod.bias.detach()
    assert lib.moco_bn_relu_maxpool_fwd_train(x.data_ptr(), y1.data_ptr(), t1.data_ptr(), N, H, W, C,
                                              _layer(w, b, m1, i1, (None, None, None, 0.1, mod.eps)),
                                              ws.data_ptr(), ws.numel(), s) == 0
    z = torch.empty_like(x)
    assert lib.moco_bn_fwd_train(x.data_ptr(), None, z.data_ptr(), N * H * W, C, w.data_ptr(), b.data_ptr(), None,
                                 None, None, 0.1, mod.eps, 1, m2.data_ptr(), i2.data_ptr(), ws.data_ptr(), ws.numel(),
                                 s) == 0
    assert lib.moco_maxpool3x3s2_fwd(z.data_ptr(), y2.data_ptr(), t2.data_ptr(), N, H, W, C, s) == 0
    torch.cuda.synchronize()
    assert torch.equal(y1, y2) and torch.equal(t1, t2) and torch.equal(m1, m2) and torch.equal(i1, i2)
    assert bool((t1 != 0).any())


@pytest.mark.parametrize("arch", ["resnet50", "resnet18"])
def test_encoder_fused_equals_the_unfused_entry_points(arch):
    """Whole encoder, forward + backward: the fused paths against the same model run on moco_bn_fwd_train /
    moco_bn_bwd / moco_maxpool3x3s2_* module by module -- bit-identical."""
    from moco_b200 import encoders, bn
    dev = torch.device("cuda:0")
    torch.manual_seed(3)
    ctor = getattr(encoders, arch)
    fused = ctor(128).to(dev).to(memory_format=torch.channels_last)
    plain = ctor(128).to(dev).to(memory_format=torch.channels_last)
    plain.load_state_dict(fused.state_dict())

    def unfused_forward(m, x):                       # the module-by-module sequence of the parent implementation
        def block(b, x):
            y = b.bn1(b.conv1(x))
            if isinstance(b, encoders._Bottleneck):
                y = b.bn2(b.conv2(y))
                last, conv = b.bn3, b.conv3
            else:
                last, conv = b.bn2, b.conv2
            r = x if b.short is None else b.short[1](b.short[0](x))
            return bn._BatchNormActFn.apply(conv(y), last.weight, last.bias, r, last.running_mean, last.running_var,
                                            last.num_batches_tracked, last.momentum, last.eps, True)
        x = m.stem[3](m.stem[1](m.stem[0](x)))
        for b in m.layers:
            x = block(b, x)
        x = torch.flatten(torch.nn.functional.adaptive_avg_pool2d(x, 1), 1)
        x = m.fc(x).float()
        return x / x.pow(2).sum(1, keepdim=True).sqrt()

    x = torch.randn(8, 3, 96, 96, device=dev).contiguous(memory_format=torch.channels_last)
    w = torch.linspace(-1, 1, 128, device=dev)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        qa = fused(x)
        qb = unfused_forward(plain, x)
    assert torch.equal(qa, qb)
    (qa * w).sum().backward()
    (qb * w).sum().backward()
    for (na, pa), (nb, pb) in zip(fused.named_parameters(), plain.named_parameters()):
        assert torch.equal(pa.grad, pb.grad), na
    for (na, ba), (nb, bb) in zip(fused.named_buffers(), plain.named_buffers()):
        assert torch.equal(ba, bb), na
