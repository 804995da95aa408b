"""moco_conv1x1_dgrad_bn_bwd + moco_bn_bwd_apply_given (csrc/conv1x1_sm90.cu, csrc/bn_nhwc.cu) against cuDNN's dgrad
followed by moco_bn_add_relu_bwd2, on the same inputs; and the autograd wiring of bn.py (_dgrad_bn_bwd) in ResNet-50
against the same model on the unfused backward."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# (C = the BatchNorm's channels = the convolution's Cin, Cout, N, H, W): every shape of ResNet-50 the fused path takes
# at batch 256, a ragged M, and two small M with one and several row chunks
SHAPES = [(256, 64, 256, 56, 56), (256, 128, 256, 56, 56), (512, 128, 256, 28, 28), (512, 256, 256, 28, 28),
          (256, 64, 3, 13, 13), (512, 256, 1, 8, 16), (1024, 64, 5, 9, 7)]


def _cl(t):
    return t.bfloat16().contiguous(memory_format=torch.channels_last)


def _f32(C, dev):
    return torch.empty(C, dtype=torch.float32, device=dev)


def _inputs(C, Cout, N, H, W, exact, seed):
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(seed)
    if exact:     # dX = dh . w is exact in any summation order: halves times {-1, 0, 1}, |dX| <= 128
        dh = _cl(torch.randint(-1, 2, (N, Cout, H, W), device=dev, generator=g) * 0.5)
        w = torch.randint(-1, 2, (Cout, C, 1, 1), device=dev, generator=g).bfloat16()
        dy2 = _cl(torch.randint(-2, 3, (N, C, H, W), device=dev, generator=g) * 0.25)
    else:
        dh = _cl(torch.randn((N, Cout, H, W), device=dev, generator=g))
        w = (torch.randn((Cout, C, 1, 1), device=dev, generator=g) * Cout ** -0.5).bfloat16()
        dy2 = _cl(torch.randn((N, C, H, W), device=dev, generator=g))
    x = _cl(torch.randn((N, C, H, W), device=dev, generator=g) * 2 + 0.5)
    mask = torch.randint(0, 256, (N * H * W, C // 8), dtype=torch.uint8, device=dev, generator=g)
    gamma = torch.rand(C, device=dev, generator=g) + 0.5
    mean = torch.randn(C, device=dev, generator=g) * 0.3 + 0.5
    invstd = torch.rand(C, device=dev, generator=g) + 0.3
    return dh, w, dy2, x, mask, gamma, mean, invstd


def _fused(dh, w, dy2, x, mask, gamma, mean, invstd):
    from moco_b200 import _lib
    from moco_b200.bn import _layer
    lib = _lib.load()
    N, C, H, W = x.shape
    M, Cout = N * H * W, w.shape[0]
    dev = x.device
    ws = torch.zeros(lib.moco_conv1x1_workspace_bytes(), dtype=torch.uint8, device=dev)
    g, dx = torch.empty_like(x), torch.empty_like(x)
    dg, db = _f32(C, dev), _f32(C, dev)
    bn = _layer(gamma, None, mean, invstd, dgamma=dg, dbeta=db)
    before = _lib.launches
    _lib.check(lib.moco_conv1x1_dgrad_bn_bwd(dh.data_ptr(), w.data_ptr(), g.data_ptr(), M, C, Cout, x.data_ptr(),
                                             mask.data_ptr(), dy2.data_ptr(), None, bn, None, ws.data_ptr(), ws.numel(),
                                             _lib.cur_stream()), "moco_conv1x1_dgrad_bn_bwd")
    _lib.check(lib.moco_bn_bwd_apply_given(g.data_ptr(), x.data_ptr(), None, M, C, bn, None, dx.data_ptr(), None,
                                           _lib.cur_stream()), "moco_bn_bwd_apply_given")
    assert _lib.launches == before + 2
    torch.cuda.synchronize()
    return g, dg, db, dx


def _unfused(dh, w, dy2, x, mask, gamma, mean, invstd):
    from moco_b200 import _lib
    from moco_b200.bn import _layer
    lib = _lib.load()
    N, C, H, W = x.shape
    M = N * H * W
    dev = x.device
    dX, _, _ = torch.ops.aten.convolution_backward(dh, x, w, None, [1, 1], [0, 0], [1, 1], False, [0, 0], 1,
                                                   [True, False, False])
    dX = dX.contiguous(memory_format=torch.channels_last)
    ws = torch.zeros(lib.moco_bn_workspace_bytes(), dtype=torch.uint8, device=dev)
    dres, dx = torch.empty_like(x), torch.empty_like(x)
    dg, db = _f32(C, dev), _f32(C, dev)
    bn = _layer(gamma, None, mean, invstd, dgamma=dg, dbeta=db)
    _lib.check(lib.moco_bn_add_relu_bwd2(dX.data_ptr(), dy2.data_ptr(), x.data_ptr(), None, mask.data_ptr(), M, C, bn,
                                         None, dx.data_ptr(), dres.data_ptr(), ws.data_ptr(), ws.numel(),
                                         _lib.cur_stream()), "moco_bn_add_relu_bwd2")
    torch.cuda.synchronize()
    return dres, dg, db, dx, dX


@pytest.mark.parametrize("C,Cout,N,H,W", SHAPES)
def test_exact_inputs_bit_identical_to_dgrad_then_bwd2(C, Cout, N, H, W):
    """With dX exact, g (= the residual gradient), dgamma, dbeta and dx equal the unfused path bit for bit; rows planted
    at the first and last row and at a tile edge each move the sums."""
    ins = list(_inputs(C, Cout, N, H, W, True, C + Cout + N))
    a, b = _fused(*ins), _unfused(*ins)[:4]
    for name, u, v in zip(("g", "dgamma", "dbeta", "dx"), a, b):
        assert torch.equal(u, v), name
    M = N * H * W
    mask = ins[4]
    for row in sorted({0, min(127, M - 1), min(128, M - 1), M - 1}):
        planted = mask.clone()
        planted[row] = 0                                   # this row's gradient is dropped
        ins2 = ins[:4] + [planted] + ins[5:]
        f2 = _fused(*ins2)
        g2, db2 = f2[0], f2[2]
        ref = _unfused(*ins2)
        assert torch.equal(g2, ref[0]) and torch.equal(db2, ref[2]), row
        moved = ref[0].permute(0, 2, 3, 1).reshape(M, C)[row] != a[0].permute(0, 2, 3, 1).reshape(M, C)[row]
        assert torch.equal(db2[moved] != b[2][moved], torch.ones_like(db2[moved], dtype=torch.bool)), row


@pytest.mark.parametrize("C,Cout,N,H,W", SHAPES[:4])
def test_seeded_inputs_against_float64_and_the_unfused_path(C, Cout, N, H, W):
    """Random inputs at batch 256: g and the sums within the bf16 + fp32-accumulation bound of float64, two calls bit
    for bit, and where g equals the unfused path's (as the forward GEMM equals cuDNN's), the sums and dx too."""
    ins = _inputs(C, Cout, N, H, W, False, 7 * C + Cout)
    dh, w, dy2, x, mask, gamma, mean, invstd = ins
    a, a2 = _fused(*ins), _fused(*ins)
    for u, v in zip(a, a2):
        assert torch.equal(u, v)
    g, dg, db, dx = a
    M = N * H * W
    rows = lambda t: t.permute(0, 2, 3, 1).reshape(M, -1)
    dX64 = rows(dh).double() @ w.view(w.shape[0], C).double()
    bits = ((mask.view(M, C // 8, 1) >> torch.arange(8, device=mask.device, dtype=torch.uint8)) & 1).view(M, C)
    g64 = (dX64 + rows(dy2).double()) * bits.double()
    err = (rows(g).double() - g64).abs()
    bound = g64.abs() * 2 ** -7 + (rows(dh).double().abs() @ w.view(w.shape[0], C).double().abs()) * 2 ** -7 + 1e-30
    assert bool((err <= bound).all()), float((err / bound).max())
    gf = rows(g).double()
    s1 = gf.sum(0)
    s2 = (gf * (rows(x).double() - mean.double())).sum(0) * invstd.double()
    # fp32 accumulation over at most a few hundred rows per thread, then fp64: 1024 ulps of the sum of magnitudes
    a2 = (gf * (rows(x).double() - mean.double())).abs().sum(0) * invstd.double()
    assert bool(((db.double() - s1).abs() <= 2 ** -14 * gf.abs().sum(0) + 2 ** -23 * s1.abs()).all())
    assert bool(((dg.double() - s2).abs() <= 2 ** -14 * a2 + 2 ** -23 * s2.abs()).all())
    ref = _unfused(*ins)
    same = torch.equal(g, ref[0])
    print(f"C={C} Cout={Cout}: g equals cuDNN dgrad + bwd2 bit for bit: {same}")
    if same:
        for name, u, v in zip(("dgamma", "dbeta", "dx"), a[1:], ref[1:4]):
            assert torch.equal(u, v), name


def _count(name):
    from moco_b200 import _lib
    lib = _lib.load()
    real = getattr(lib, name)
    calls = [0]

    def counted(*args):
        calls[0] += 1
        return real(*args)

    setattr(lib, name, counted)
    return calls, lambda: setattr(lib, name, real)


def test_resnet50_autograd_under_autocast(monkeypatch):
    """ResNet-50 at 16 x 224^2 under bf16 autocast with the shape gate lifted: one fused call per conv1 fed by an
    identity block's output (stride-1 table shapes), the same total of library launches as the unfused backward,
    gradients no further from fp32 than the unfused path's (the bound of test_gpu_conv1x1), and a second backward
    through the retained graph equal to the first."""
    from moco_b200 import _lib, bn, encoders
    dev = torch.device("cuda:0")
    torch.manual_seed(11)
    models = [encoders.resnet50(128).to(dev).to(memory_format=torch.channels_last) for _ in range(3)]
    for m in models[1:]:
        m.load_state_dict(models[0].state_dict())
    x = torch.randn(16, 3, 224, 224, device=dev).contiguous(memory_format=torch.channels_last)
    wv = torch.linspace(-1, 1, 128, device=dev)
    monkeypatch.setattr(bn, "_conv1x1_wins", lambda M, Cin, Cout: True)
    blocks = models[0].layers
    expected = sum(1 for i in range(1, len(blocks)) if blocks[i - 1].short is None)
    out = {}

    def step(m, key, autocast=True, twice=False):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            q = m(x)
        loss = (q * wv).sum()
        loss.backward(retain_graph=twice)
        grads = [p.grad.float().clone() for p in (m.fc.weight, m.stem[0].weight, m.layers[1].conv1.weight,
                                                  m.layers[1].bn3.weight)]
        if twice:
            for p in m.parameters():
                p.grad = None
            loss.backward()
            again = [p.grad.float() for p in (m.fc.weight, m.stem[0].weight, m.layers[1].conv1.weight,
                                              m.layers[1].bn3.weight)]
            for u, v in zip(grads, again):
                assert torch.equal(u, v)
        out[key] = grads

    step(models[2], "fp32", autocast=False)
    monkeypatch.setattr(bn, "_dgrad_wins", lambda M, Cin, Cout: True)
    calls, undo = _count("moco_conv1x1_dgrad_bn_bwd")
    try:
        before = _lib.launches
        step(models[0], "new", twice=True)
        launches_a = (_lib.launches - before)
    finally:
        undo()
    assert calls[0] == 2 * expected, (calls[0], expected)
    monkeypatch.setattr(bn, "_dgrad_wins", lambda M, Cin, Cout: False)
    before = _lib.launches
    step(models[1], "old", twice=True)
    launches_b = _lib.launches - before
    assert launches_a == launches_b
    for i, name in enumerate(("fc", "stem", "conv1", "bn3")):
        ref = out["fp32"][i]
        e_new = float((out["new"][i] - ref).norm() / ref.norm())
        e_old = float((out["old"][i] - ref).norm() / ref.norm())
        assert e_new < max(2.0 * e_old, 0.05), (name, e_new, e_old)


def test_fallbacks(monkeypatch):
    """An extra consumer of a block output makes the producer take its full backward on what it receives (g plus the
    other gradient): close to the unfused path's gradients.  set_fused(False) never reaches the fused call."""
    from moco_b200 import bn, encoders
    dev = torch.device("cuda:0")
    torch.manual_seed(3)
    stage = torch.nn.Sequential(encoders._Bottleneck(64, 64, 1), encoders._Bottleneck(256, 64, 1),
                                encoders._Bottleneck(256, 64, 1)).to(dev).to(memory_format=torch.channels_last)
    x0 = torch.randn(4, 64, 32, 32, device=dev).contiguous(memory_format=torch.channels_last)
    monkeypatch.setattr(bn, "_conv1x1_wins", lambda M, Cin, Cout: True)

    def grads(wins):
        monkeypatch.setattr(bn, "_dgrad_wins", lambda M, Cin, Cout: wins)
        stage.zero_grad(set_to_none=True)
        x = x0.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            h = stage[1](stage[0](x))                     # an identity block's output: stage[2].conv1 fuses
            y = stage[2](h)
            loss = y.float().square().mean() + h.float().sum() * 1e-3      # h: an extra consumer
        loss.backward()
        return [x.grad.float()] + [p.grad.float() for p in stage.parameters()]

    calls, undo = _count("moco_conv1x1_dgrad_bn_bwd")
    try:
        a, b = grads(True), grads(False)
        assert calls[0] == 1
        for u, v in zip(a, b):
            assert float((u - v).norm()) <= 0.02 * float(v.norm()) + 1e-6
        bn.set_fused(False)
        try:
            grads(True)
        finally:
            bn.set_fused(True)
        assert calls[0] == 1
    finally:
        undo()


def test_cur_stream_is_the_current_stream():
    """_lib.cur_stream (the raw handle every launch is enqueued on) is torch's current stream, also inside a side
    stream and on a second device when there is one."""
    from moco_b200 import _lib
    assert _lib.cur_stream() == torch.cuda.current_stream().cuda_stream
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        assert _lib.cur_stream() == side.cuda_stream != torch.cuda.default_stream().cuda_stream
    if torch.cuda.device_count() > 1:
        with torch.cuda.device(1):
            assert _lib.cur_stream() == torch.cuda.current_stream(1).cuda_stream
