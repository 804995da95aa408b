"""moco_conv1x1_bn_stats (csrc/conv1x1_sm90.cu) over the whole envelope include/moco_b200.h promises, against an exact
reference that shares no code with the kernel; and moco_bn_fwd_train's statistics, the other caller of bn_reduce.cuh,
at ResNet-50's batch-256 BatchNorm shapes against the same reference.

Exact-arithmetic inputs.  x is in {-1, 0, 1}; weight row c is +1 in column 0 and s_c = +-1 in one column j_c >= 1.
Every y = x[:, 0] + s_c x[:, j_c] is an integer in [-2, 2] and must equal that gather bit for bit.  Every d = y - y[0, c]
is an integer in [-4, 4], so each fp32 sum of d and d^2 the kernel forms (per thread, per warp, per CTA) is exact while
a CTA's row chunk has fewer than 2^24 / 16 rows, which is asserted from the plan (_plan).  The fp64 totals are then the
exact integers S1 = sum d and S2 = sum d^2 in any order, and mean, invstd and the running statistics are fixed by the
IEEE operations of bn_stats_channel (bn_reduce.cuh), which _channel_stats performs one at a time.  The statistics are
computed from the y the kernel stored, after y is checked, so that a wrong y is reported as one.

Planted rows.  Row 0 is -1 in every channel (the shift) and the planted rows are +1 (d = 2): the first and last row of
every CTA row chunk, both sides of the 128-row tile boundaries next to the chunk edges, the ragged last tile and row
M - 1.  A CTA that loses or repeats one of them moves S1 by 2, and a CTA that takes its shift from its own first tile
(a planted row) instead of row 0 moves S1 by 2 per row of its chunk.  Each case asserts that such a change moves mean
or invstd in every channel, so the comparison can fail.

Size: the largest cases hold one 6.6 GB operand (802,816 rows x 4096 channels of bf16: byte offsets past 2^32) and
stay under 10 GB of device memory."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

gpu = pytest.mark.gpu

COUTS = [64, 128, 192, 320, 384, 2048, 4096]       # BN = 64 and 128; 1 .. 32 column slices; 1 .. 64 slabs
CINS = [64, 192, 1088, 4096]                      # 1, 3, 17 and 64 K chunks
SMALL_M = [1, 31, 32, 127, 128, 129, 255, 256, 257, 258]   # the 128-row tile and the 256-row statistics chunk


def _plan(M, C, unroll=8):
    """bn_reduce_plan (csrc/bn_nhwc.cu) with 2 CTAs per SM and kBnSms = 132, as bn_stats_plan calls it (unroll 8) or
    bn_bwd_reduce_plan (unroll 4): the passes of 32 rows, the passes of each CTA's row chunk and R, the CTAs per
    64-channel slab."""
    passes = -(-M // 32)
    r = max(1, min(132 * 2 // (C // 64), -(-passes // unroll)))
    per = -(-passes // r)
    per = -(-per // unroll) * unroll
    return passes, per, -(-passes // per)


def _r_changes(C, limit, unroll=8):
    """The row counts M <= limit at which the plan's R differs from its value at M - 1 (M = 1 first)."""
    out, prev = [], None
    for p in range(1, -(-limit // 32) + 1):
        R = _plan(32 * p, C, unroll)[2]
        if R != prev:
            out.append(32 * p - 31)
            prev = R
    return out


def _planted(M, C, unroll=8):
    """The planted rows of an M-row case with C channels (row 0 excluded: it holds the shift)."""
    _, per, R = _plan(M, C, unroll)
    L = 32 * per
    rows = set()
    for k in range(R):
        s, e = k * L, min((k + 1) * L, M)
        rows |= {s - 1, s, s + 127, s + 128, e - 1}
        if e < M:
            rows |= {e - 129, e - 128}
    t = (M - 1) // 128 * 128                    # the last tile, ragged unless M is a multiple of 128
    rows |= {t - 1, t, (t + M - 1) // 2, M - 1}
    return sorted(r for r in rows if 0 < r < M)


def _round(q, bits):
    """The rational q rounded to the nearest number of `bits` significant bits, ties to even (normal range only)."""
    q = Fraction(q)
    if q == 0:
        return q
    a = abs(q)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if a < Fraction(2) ** e:
        e -= 1
    scale = Fraction(2) ** (bits - 1 - e)
    n, rem = divmod(a * scale, 1)
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and n % 2 == 1):
        n += 1
    return n / scale if q > 0 else -n / scale


def _f64(q):
    return float(_round(q, 53))


def _f32(q):
    return np.float32(float(_round(q, 24)))


def _q(v):
    return Fraction(float(v))


def _channel_stats(s1, s2, shift, M, eps, momentum, rm=None, rv=None):
    """bn_stats_channel (csrc/bn_reduce.cuh) on the exact totals s1, s2 (ints), one IEEE operation at a time.

    The contractions are those of the SASS nvcc 12.9 builds from it (-O3, default -fmad=true; read with
    cuobjdump -sass) in all three kernels that inline it (bn_stats_kernel and conv1x1_stats_kernel<64/128>): two FMAs,
    var = fma(s2, inv_m, -(md * md)) and running = fma(momentum, new, running * (1 - momentum)); shift + md is a DADD,
    and the sqrt and both divisions are correctly rounded.  Python floats are IEEE doubles with correctly rounded
    +, -, *, / and sqrt; each fused operation is evaluated exactly in Fraction and rounded once.
    Returns float32 (mean, invstd, running_mean, running_var), the last two None without running statistics."""
    inv_m = 1.0 / M
    md = s1 * inv_m
    var = max(_f64(Fraction(s2) * _q(inv_m) - _q(md * md)), 0.0)
    mean = np.float32(shift + md)
    invstd = np.float32(1.0 / math.sqrt(var + float(np.float32(eps))))
    if rm is None:
        return mean, invstd, None, None
    m = np.float32(momentum)
    keep = np.float32(1.0) - m
    unbiased = var * (M / (M - 1)) if M > 1 else var
    rm = _f32(_q(m) * _q(mean) + _q(np.float32(rm) * keep))
    rv = _f32(_q(m) * _q(np.float32(unbiased)) + _q(np.float32(rv) * keep))
    return mean, invstd, rm, rv


def _totals(y, ref=None):
    """(shift y[0, c], S1, S2) of y [M, C] as Python lists, exactly; ref(i, n), when given, is the exact value of rows
    i .. i + n - 1, which y must equal bit for bit."""
    M, C = y.shape
    step = min(2 ** 19, 2 ** 27 // C)           # fp32 column sums of at most 2^19 rows of d^2 <= 16: exact
    shift = y[0].float()
    s1 = torch.zeros(C, dtype=torch.float64, device=y.device)
    s2 = torch.zeros_like(s1)
    for i in range(0, M, step):
        yc = y[i:i + step].float()
        if ref is not None:
            r = ref(i, yc.shape[0])
            if not torch.equal(yc, r):
                bad = (yc != r).nonzero()[0].tolist()
                raise AssertionError(f"y[{i + bad[0]}, {bad[1]}] = {float(yc[tuple(bad)])}, exact {float(r[tuple(bad)])}")
        d = yc - shift
        s1 += d.sum(0).double()
        s2 += (d * d).sum(0).double()
    return shift.tolist(), [int(v) for v in s1.tolist()], [int(v) for v in s2.tolist()]


def _expect(totals, M, momentum, eps, before):
    """Expected (mean, invstd, running_mean, running_var) as float32 arrays from _totals and the running statistics
    before the call (None: without)."""
    shift, s1, s2 = totals
    rm = rv = [None] * len(s1)
    if before is not None:
        rm, rv = before[0].tolist(), before[1].tolist()
    out = [_channel_stats(a, b, h, M, eps, momentum, m, v) for a, b, h, m, v in zip(s1, s2, shift, rm, rv)]
    return [None if out[0][k] is None else np.array([o[k] for o in out], dtype=np.float32) for k in range(4)]


def _assert_equal(name, got, want):
    got = got.cpu().numpy()
    if not np.array_equal(got, want):
        c = int(np.nonzero(got != want)[0][0])
        raise AssertionError(f"{name}[{c}] = {got[c]!r}, exact {want[c]!r} ({int((got != want).sum())} channels differ)")


def _assert_sensitive(totals, dp, M, momentum, eps, want):
    """Dropping or repeating one planted row (d = dp in every channel) changes mean or invstd of every channel."""
    shift, s1, s2 = totals
    for sign in (-1, 1):
        for c, (a, b, h) in enumerate(zip(s1, s2, shift)):
            mean, invstd, _, _ = _channel_stats(a + sign * dp, b + sign * dp * dp, h, M, eps, momentum)
            assert mean != want[0][c] or invstd != want[1][c], ("a planted row would go unseen", c, sign)


def _check_stats(totals, M, C, momentum, eps, before, after, mean, invstd, dp):
    """mean, invstd and the running statistics `after` the call against the emulation; nbt advanced by one."""
    _, per, _ = _plan(M, C)
    assert 16 * 32 * per < 2 ** 24, "a CTA partial could round"
    want = _expect(totals, M, momentum, eps, before)
    _assert_equal("mean", mean, want[0])
    _assert_equal("invstd", invstd, want[1])
    if before is not None:
        _assert_equal("running_mean", after[0], want[2])
        _assert_equal("running_var", after[1], want[3])
        if before[2] is not None:
            assert int(after[2]) == int(before[2]) + 1
    if M > 1:
        _assert_sensitive(totals, dp, M, momentum, eps, want)


# ---- the convolution

def _weights(Cin, Cout, g):
    """(w [Cout, Cin] bf16, j, s): +1 in column 0 and s_c in column j_c of row c; j covers the second and the last K
    chunk."""
    dev = g.device
    j = torch.randint(1, Cin, (Cout,), device=dev, generator=g)
    j[-1] = Cin - 1
    if Cin > 64:
        j[0] = 64
    s = (torch.randint(0, 2, (Cout,), device=dev, generator=g) * 2 - 1).float()
    w = torch.zeros(Cout, Cin, device=dev)
    w[:, 0] = 1
    w[torch.arange(Cout, device=dev), j] = s
    return w.to(torch.bfloat16), j, s


def _fill_x(x, g, planted):
    """x [M, Cin] in {-1, 0, 1}, row 0 = -e_0 (y[0, c] = -1), the planted rows = e_0 (y = 1)."""
    M, Cin = x.shape
    step = max(1, 2 ** 28 // Cin)
    for i in range(0, M, step):
        n = min(step, M - i)
        x[i:i + n] = torch.randint(-1, 2, (n, Cin), device=x.device, generator=g, dtype=torch.int8)
    x[0] = 0
    x[0, 0] = -1
    if planted:
        p = torch.tensor(planted, device=x.device)
        x[p] = 0
        x[p, 0] = 1
    return x


def _new_ws(dev):
    from moco_b200 import _lib
    return torch.zeros(_lib.load().moco_conv1x1_workspace_bytes(), dtype=torch.uint8, device=dev)


def _launch(x, w, y, mean, invstd, stats, momentum, eps, ws):
    from moco_b200 import _lib
    from moco_b200.bn import _layer
    rm, rv, nbt = stats if stats is not None else (None, None, None)
    _lib.check(_lib.load().moco_conv1x1_bn_stats(
        x.data_ptr(), w.data_ptr(), y.data_ptr(), x.shape[0], x.shape[1], w.shape[0],
        _layer(None, None, mean, invstd, (rm, rv, nbt, momentum, eps)), ws.data_ptr(), ws.numel(), _lib.cur_stream()),
        "moco_conv1x1_bn_stats")


def _running(C, dev, g, mode="full"):
    """(running_mean, running_var, num_batches_tracked) for mode full, no_nbt (nbt None) or none (None)."""
    if mode == "none":
        return None
    rm = torch.randn(C, device=dev, generator=g)
    rv = torch.rand(C, device=dev, generator=g) + 0.5
    return rm, rv, (torch.tensor(7, dtype=torch.long, device=dev) if mode == "full" else None)


def _snapshot(stats):
    return None if stats is None else tuple(None if t is None else t.clone() for t in stats)


class _Case:
    """One shape's inputs and outputs on cuda:0."""

    def __init__(self, Cin, Cout, M, seed, stats="full"):
        dev = torch.device("cuda:0")
        self.g = torch.Generator(device=dev).manual_seed(seed)
        self.M, self.Cin, self.Cout = M, Cin, Cout
        self.planted = _planted(M, Cout)
        self.x = _fill_x(torch.empty(M, Cin, dtype=torch.bfloat16, device=dev), self.g, self.planted)
        self.w, self.j, self.s = _weights(Cin, Cout, self.g)
        self.y = torch.empty(M, Cout, dtype=torch.bfloat16, device=dev)
        self.mean = torch.empty(Cout, device=dev)
        self.invstd = torch.empty(Cout, device=dev)
        self.stats = _running(Cout, dev, self.g, stats)

    def exact(self, i, n):
        xc = self.x[i:i + n]
        return xc[:, :1].float() + xc[:, self.j].float() * self.s

    def run(self, momentum=0.1, eps=1e-5, ws=None):
        before = _snapshot(self.stats)
        _launch(self.x, self.w, self.y, self.mean, self.invstd, self.stats, momentum, eps,
                ws if ws is not None else _new_ws(self.x.device))
        self.check(before, momentum, eps)

    def check(self, before, momentum, eps):
        totals = _totals(self.y, self.exact)
        _check_stats(totals, self.M, self.Cout, momentum, eps, before, self.stats, self.mean, self.invstd, 2)


def _cases():
    out = []
    for a, M in enumerate(SMALL_M):
        for b, Cout in enumerate(COUTS):
            out.append((CINS[(a + b) % len(CINS)], Cout, M))
    for b, Cout in enumerate(COUTS):
        ch = _r_changes(Cout, 802816)
        rs = [_plan(m, Cout)[2] for m in ch]
        top = rs.index(max(rs))
        picks = ch[top:top + 2] + (ch[-1:] if Cout in (64, 192) else [])     # R reaches its maximum, then drops
        out += [(CINS[(b + k) % 2], Cout, m + k) for m in picks for k in (-1, 0, 1)]
    out += [
        (1088, 192, 50176),      # the dispatch threshold: BN = 64, three slices, 17 K chunks
        (4096, 2048, 50176),
        (256, 64, 802816),       # batch 256 at 56^2
        (64, 4096, 802816),      # y is 6.6 GB (offsets past 2^32); 64 slabs
        (4096, 320, 802816),     # x is 6.6 GB; BN = 64, five slices
        (65536, 64, 257),        # 1024 K chunks: the ring wraps hundreds of times per tile
        (65536, 384, 1000),
    ]
    return out


@gpu
@pytest.mark.parametrize("Cin,Cout,M", _cases())
def test_envelope_exact(Cin, Cout, M):
    """y bit-identical to the exact product; mean, invstd, the running statistics and num_batches_tracked exactly
    bn_stats_channel's on the exact sums of the y stored."""
    case = _Case(Cin, Cout, M, seed=M * 7 + Cin * 3 + Cout)
    case.run()
    if M * max(Cin, Cout) * 2 > 2 ** 32:
        del case
        torch.cuda.empty_cache()


@gpu
@pytest.mark.parametrize("momentum,eps", [(0.1, 1e-5), (0.01, 1e-3)])
@pytest.mark.parametrize("mode", ["full", "no_nbt", "none"])
@pytest.mark.parametrize("Cin,Cout,M", [(192, 320, 13313), (64, 4096, 1025)])
def test_running_statistics(Cin, Cout, M, mode, momentum, eps):
    """Null running statistics, a null num_batches_tracked and two (momentum, eps) pairs."""
    case = _Case(Cin, Cout, M, seed=M + Cout, stats=mode)
    case.run(momentum, eps)


@gpu
def test_one_workspace_across_slab_counts():
    """Cout = 4096 (64 slabs, 4 CTAs each), 64 (1 slab, 196 CTAs), 4096 again on one workspace: every slab's ticket
    counter is re-armed for the next call, and each call matches its own reference."""
    ws = _new_ws(torch.device("cuda:0"))
    for k, Cout in enumerate((4096, 64, 4096)):
        _Case(256, Cout, 50176, seed=40 + k).run(ws=ws)


@gpu
def test_graph_replay():
    """One call captured in a CUDA graph and replayed three times on new inputs: each replay's y and statistics match
    the reference, and num_batches_tracked advances by three."""
    case = _Case(192, 320, 20000, seed=77)
    ws = _new_ws(case.x.device)
    case.run(ws=ws)                                  # warm-up: the kernel attributes are set outside the capture
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _launch(case.x, case.w, case.y, case.mean, case.invstd, case.stats, 0.1, 1e-5, ws)
    nbt0 = int(case.stats[2])
    for _ in range(3):
        _fill_x(case.x, case.g, case.planted)
        before = _snapshot(case.stats)
        graph.replay()
        torch.cuda.synchronize()
        case.check(before, 0.1, 1e-5)
    assert int(case.stats[2]) == nbt0 + 3


# ---- moco_bn_fwd_train, the statistics pass

# (M, C) of ResNet-50's training BatchNorms at batch 256 (stem; stages 1-4 at 56^2, 28^2, 14^2, 7^2)
BN_SHAPES = [(3211264, 64), (802816, 64), (802816, 128), (802816, 256), (200704, 128), (200704, 256), (200704, 512),
             (50176, 256), (50176, 512), (50176, 1024), (12544, 512), (12544, 2048)]


@gpu
@pytest.mark.parametrize("M,C", BN_SHAPES)
def test_bn_fwd_train_statistics_exact(M, C):
    """moco_bn_fwd_train's mean, invstd and running statistics exactly bn_stats_channel's on the exact sums: x in
    {-2, .., 2}, row 0 = -2 and the planted rows +2 (d = 4).  Its output is not checked here."""
    from moco_b200 import _lib
    from moco_b200.bn import _workspace
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(M + C)
    x = torch.randint(-2, 3, (M, C), device=dev, generator=g, dtype=torch.int8).to(torch.bfloat16)
    x[0] = -2
    x[torch.tensor(_planted(M, C), device=dev)] = 2
    stats = _running(C, dev, g)
    before = _snapshot(stats)
    mean, invstd = torch.empty(C, device=dev), torch.empty(C, device=dev)
    gamma, beta = torch.ones(C, device=dev), torch.zeros(C, device=dev)
    z = torch.empty_like(x)
    ws = _workspace(dev)
    _lib.check(_lib.load().moco_bn_fwd_train(
        x.data_ptr(), None, z.data_ptr(), M, C, gamma.data_ptr(), beta.data_ptr(), stats[0].data_ptr(),
        stats[1].data_ptr(), stats[2].data_ptr(), 0.1, 1e-5, 1, mean.data_ptr(), invstd.data_ptr(), ws.data_ptr(),
        ws.numel(), _lib.cur_stream()), "moco_bn_fwd_train")
    _check_stats(_totals(x), M, C, 0.1, 1e-5, before, stats, mean, invstd, 4)


# ---- the reference helpers, by hand (no GPU)

def test_reference_helpers_by_hand():
    """_plan, _round and _channel_stats on cases computed by hand."""
    assert _plan(257, 64) == (9, 8, 2)                   # 256-row chunks while R < 264 / slabs
    assert _plan(67585, 64) == (2113, 16, 133)           # ceil(2113 / 264) = 9 -> 16 passes: R drops from 264
    assert _plan(802816, 4096) == (25088, 6272, 4)       # 64 slabs: 4 CTAs each
    assert _r_changes(4096, 1100) == [1, 257, 513, 769, 1025]
    assert _planted(300, 64) == [127, 128, 255, 256, 277, 299]   # chunks [0, 256), [256, 300)
    # ties to even at 24 bits; 1/3 to the nearest float32
    assert _round(2 ** 24 + 1, 24) == 2 ** 24 and _round(2 ** 24 + 3, 24) == 2 ** 24 + 4
    assert _f32(Fraction(-1, 3)) == np.float32(-1.0 / 3.0)
    # a fused fp32 update keeps the product's low bits: (1 + 2^-23)^2 - (1 + 2^-22) = 2^-46, where fl(a * b) - c = 0
    a = 1 + 2.0 ** -23
    assert _f32(_q(a) * _q(a) - _q(1 + 2.0 ** -22)) == np.float32(2.0 ** -46)
    b = 1 + 2.0 ** -52                                   # and in double: 2^-104, where fl(b * b) - c = 0
    assert _f64(_q(b) * _q(b) - _q(1 + 2.0 ** -51)) == 2.0 ** -104
    # y = -1, 1, 1, -1: shift -1, S1 = 4, S2 = 8; md = 1, var = 2 - 1 = 1, unbiased 4/3; eps = 0.25, momentum 0.5
    mean, invstd, rm, rv = _channel_stats(4, 8, -1.0, 4, 0.25, 0.5, 0.0, 1.0)
    assert mean == np.float32(0.0) and invstd == np.float32(1.0 / math.sqrt(1.25))
    # rv = 0.5 + 0.5 * f32(4/3) = (2^23 + 11184811) 2^-24: 25 bits, a tie, rounded to even 9786710 2^-23
    assert rm == np.float32(0.0) and rv == np.float32(9786710 * 2.0 ** -23)
