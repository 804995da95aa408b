"""The training BatchNorm passes of csrc/bn_nhwc.cu that no other exact test reaches, against exact references that
share no code with them: moco_bn_bwd in every mask mode (the stem's, bn1's and bn2's backward), the downsample blocks'
backward with the shortcut BN (moco_bn_add_relu_bwd / _bwd2: bn3 and the shortcut BN on one g), the apply without a
residual (moco_bn_fwd_train_given, moco_bn_fwd_train's output) and the stem's BatchNorm + ReLU + max pool
(moco_bn_relu_maxpool_fwd_train) chained with its backward (moco_maxpool3x3s2_bwd, then moco_bn_bwd).  Every output
is compared exactly (torch.equal / np.array_equal on values).

Inputs.  dy (and dy2) on a 1/4 grid in [-2, 2]; x and the given save_mean on a common 1/8 grid, |x - mean| <= 8, with
the sign of the gradient, so that S2 outgrows fp32 while each CTA's partials stay exact; the shortcut's x2 and mean2
the same, with random signs.  gamma (both signs), invstd and the shortcut's gamma2, invstd2 are arbitrary floats and
beta = |gamma invstd| (1 + u), u in [0, 1), so that the planted rows' ReLU is on.  Channel 1 has gamma = 1e-42 and
beta = 0: every pre-activation z = fmaf(x, ca, cb) is a positive or negative subnormal below 2^-134, which bf16
stores as zero.  Channel 2 has beta = -1e4: all zeros.  Channel 3 has ca = 2^-136 and beta = 0: z = (x - mean) 2^-136
exactly, which bf16 rounds to zero up to x - mean = 4, the tie at 2^-134 included, and to 2^-133 or more above.

The ReLU mask is y > 0 of the output as the forward stores it,
    ca = gamma * invstd,  cb = fmaf(-mean, ca, beta),  y = bf16(max(fp32(fmaf(x, ca, cb) + r), 0))   (r = 0 or the
residual), so the mask moco_bn_bwd recomputes from x must be the mask bits (relu_bits) and the y of
moco_bn_fwd_train_given on the same x, which is checked against the same formula.  Then, with g = mask . dy (or
mask . bf16(dy + dy2)) and S1 = sum g, S2 = sum g (x - mean), S3 = sum g (x2 - mean2) exact in float64,
    dbeta = fp32(S1),  dgamma = fp32(S2 * invstd),   the shortcut's dbeta = dbeta, its dgamma = fp32(S3 * invstd2),
    dx = bf16(fmaf(cA, g, fmaf(cB, x, cD))) with bwd_coefs(gamma, mean, invstd, dbeta, dgamma),
    dresidual = g, or with the shortcut BN bf16(fmaf(cA2, g, fmaf(cB2, x2, cD2))) with
                bwd_coefs(gamma2, mean2, invstd2, dbeta, the shortcut's dgamma).
That no fp32 partial can round is asserted per CTA row chunk of bn_bwd_reduce_plan (_plan with unroll 4) from the
data.  Planted rows (g = 2, x - mean = x2 - mean2 = 1, mask on) at the chunk and tile edges must each move dbeta or
dgamma, when dropped or repeated, in every channel whose planted mask is on (all but channels 1 to 3).  A few rows of
the two-gradient cases round in bf16(dy + dy2), ties included: dy in 256 .. 4096, dy2 in +-{1/4, 1/2, 1}, with
x - mean = x2 - mean2 = +-1/8.

The stem.  x on a 1/2 grid in [-1.5, 1.5] (ties in every window) with the call's own statistics: y and the tap bytes
are _pool_reference of the exact BatchNorm + ReLU values.  Its backward takes given statistics on the 1/8 grid, so that
its sums are exact: g of moco_maxpool3x3s2_bwd equals _pool_bwd_reference, then moco_bn_bwd's outputs equal the
reference above.

Contractions.  cuobjdump -sass of the library nvcc 12.9 builds (-O3, default -fmad=true) shows only the source's
explicit fmaf in the instances these tests run: per channel one FMUL and one FFMA for ca / cb, bwd_coefs' six FMUL and
one FFMA; per element one FFMA in bn_apply_kernel and for the mask from x, one per sum in the reduction, and the two
FFMA of dx (and of the shortcut's dx2).

Size.  The largest cases are ResNet-50's at batch 256: the stem's 3,211,264 x 64 (411 MB per tensor) and the first
downsample block's 802,816 x 256 with six such tensors.  Every case stays under 10 GB of device memory (asserted)."""
import types

import numpy as np
import pytest
import torch

from tests.test_gpu_conv1x1_envelope import BN_SHAPES, _assert_equal, _plan, _planted, _r_changes, _running
from tests.test_gpu_conv1x1_fused_envelope import (RESIDUAL_BN, _Bn, _bits, _bwd_coefs, _equal, _fma32, _fmaf, _pack,
                                                   _rows, memory)  # noqa: F401  (memory: the fixture)
from tests.test_gpu_junction import _pool_bwd_reference, _pool_reference

gpu = pytest.mark.gpu
STATS_GIVEN = 1                              # MOCO_BN_STATS_GIVEN
UNDERFLOW, ZEROS, TIE = 1, 2, 3             # channels: gamma = 1e-42, beta = 0; beta = -1e4; ca = 2^-136, beta = 0

CS = [64, 128, 256, 512, 1024, 2048]
SMALL_M = [1, 2, 31, 32, 33, 127, 128, 129, 255, 256, 257]
# vectors of 16 bytes one grid-stride trip of an element-wise kernel covers at its largest grid: kBnThreads x unroll x
# kBnSms x CTAs per SM -- bn_apply_kernel<8, 2>, bn_bwd_apply_kernel<2, 3> (moco_bn_bwd, moco_bn_add_relu_bwd without
# a shortcut) and <2, 2> (with the shortcut BN or a second gradient)
TRIP_FWD, TRIP_BWD, TRIP_SC = 256 * 8 * 264, 256 * 2 * 396, 256 * 2 * 264


def _lib():
    from moco_b200 import _lib as L
    return L


def _ws(dev):
    return torch.zeros(_lib().load().moco_bn_workspace_bytes(), dtype=torch.uint8, device=dev)


def _apply_grid(V, unroll, ctas):
    """bn_apply_grid (csrc/bn_nhwc.cu) with kBnSms = 132: CTAs of the element-wise kernels for V vectors."""
    return max(1, min(-(-V // (256 * unroll)), 132 * ctas))


def _r_edges(C):
    """M - 1, M, M + 1 where the backward reduction's R reaches its maximum and where it first drops, as the fused
    envelope picks them."""
    ch = _r_changes(C, 802816, 4)
    rs = [_plan(m, C, 4)[2] for m in ch]
    top = rs.index(max(rs))
    return [m + k for m in ch[top:top + 2] for k in (-1, 0, 1) if m + k >= 1]


def _trip_edges(trip):
    """(C, M) with V = M C / 8 one row short of, at, and one row past one or two whole trips."""
    return [(C, k * trip * 8 // C + d) for C, k in ((64, 1), (2048, 1), (256, 2)) for d in (-1, 0, 1)]


def _y_ref(x, ca, cb, r, relu):
    """bn_apply_kernel's y = bf16(relu?(fp32(fmaf(x, ca, cb) + r))), r = 0 without a residual."""
    z = _fma32(x.float(), ca, cb) + (r.float() if r is not None else 0.0)
    if relu:
        z = torch.maximum(z, torch.zeros_like(z))
    return z.bfloat16()


class _Params:
    """One BatchNorm's gamma, beta and given statistics (module docstring), and bn_apply_kernel's ca, cb."""

    def __init__(self, C, g, dev):
        self.gamma = torch.randn(C, device=dev, generator=g)
        self.invstd = torch.rand(C, device=dev, generator=g) + 0.3
        self.mean = torch.randint(-8, 9, (C,), device=dev, generator=g) / 8.0
        self.beta = (self.gamma * self.invstd).abs() * (1 + torch.rand(C, device=dev, generator=g))
        self.gamma[UNDERFLOW] = 1e-42
        self.beta[UNDERFLOW] = 0.0
        self.beta[ZEROS] = -1e4
        self.gamma[TIE], self.invstd[TIE], self.beta[TIE] = 2.0 ** -136, 1.0, 0.0
        self.ca, self.cb = _Bn.coefs(self)

    def layer(self, dgamma=None, dbeta=None):
        from moco_b200.bn import _layer
        return _layer(self.gamma, self.beta, self.mean, self.invstd, (None, None, None, 0.1, 1e-5), dgamma, dbeta)


# kinds of backward: moco_bn_bwd with relu, has_residual = (1, 0) "x", (1, 1) "y", (0, 0) "none", (0, 1) "none_res";
# moco_bn_add_relu_bwd without a shortcut BN "bits", with one "sc"; moco_bn_add_relu_bwd2 with one "sc2"
BWD_KINDS = ["x", "y", "none", "none_res"]
SC_KINDS = ["sc2", "sc", "bits"]


class _Bwd:
    """One backward case on cuda:0.  given = (params, dy, x): the stem's chained backward, no planted rows."""

    def __init__(self, M, C, kind, seed, given=None):
        dev = torch.device("cuda:0")
        self.M, self.C, self.kind = M, C, kind
        self.g = torch.Generator(device=dev).manual_seed(seed)
        self.sc = _Params(C, self.g, dev) if kind in ("sc", "sc2") else None
        new = lambda: torch.empty(M, C, dtype=torch.bfloat16, device=dev)
        self.dy2 = new() if kind == "sc2" else None
        self.x2 = new() if self.sc is not None else None
        self.mask = torch.empty(M, C // 8, dtype=torch.uint8, device=dev) if kind in SC_KINDS else None
        if kind in ("x", "y"):                       # the forward's output and mask bits on the same x
            self.y, self.ybits = new(), torch.empty(M, C // 8, dtype=torch.uint8, device=dev)
        _, per, self.R = _plan(M, C, 4)
        self.L = 32 * per                            # rows per CTA chunk
        if given is None:
            self.p = _Params(C, self.g, dev)
            self.dy, self.x = new(), new()
            self.planted = sorted(set(_planted(M, C, 4)) | {0})
            cand = [M // 5, 2 * M // 5, M // 2 + 1, 3 * M // 5, 4 * M // 5, M - 2] if self.dy2 is not None else []
            self.rounding = sorted({r for r in cand if 0 <= r < M} - set(self.planted))
            self.fill()
        else:
            self.p, self.dy, self.x = given
            self.planted, self.rounding = [], []
        self.dx = new()
        self.dres = new() if kind in ("y", "none_res", "bits", "sc", "sc2") else None
        self.dgamma, self.dbeta = torch.empty(C, device=dev), torch.empty(C, device=dev)
        if self.sc is not None:
            self.sc_dgamma, self.sc_dbeta = torch.empty(C, device=dev), torch.empty(C, device=dev)

    def fill(self):
        """New inputs in place (graph replays read the same buffers)."""
        M, C, g, dev, p, s = self.M, self.C, self.g, self.x.device, self.p, self.sc
        for i in range(0, M, _rows(C)):
            n = min(_rows(C), M - i)
            dy = torch.randint(-8, 9, (n, C), device=dev, generator=g, dtype=torch.int8) / 4.0
            self.dy[i:i + n] = dy
            if self.dy2 is not None:
                self.dy2[i:i + n] = torch.randint(-8, 9, (n, C), device=dev, generator=g, dtype=torch.int8) / 4.0
                dy = dy + self.dy2[i:i + n].float()
            d = torch.randint(0, 65, (n, C), device=dev, generator=g, dtype=torch.int8) / 8.0
            self.x[i:i + n] = p.mean + d * torch.sign(dy)
            if s is not None:
                self.x2[i:i + n] = s.mean + torch.randint(-64, 65, (n, C), device=dev, generator=g, dtype=torch.int8) / 8.0
            if self.mask is not None:
                self.mask[i:i + n] = torch.randint(0, 256, (n, C // 8), device=dev, generator=g, dtype=torch.uint8)
        q = torch.tensor(self.planted, device=dev)
        self.dy[q] = 2.0 if self.dy2 is None else 1.0           # g = 2
        if self.dy2 is not None:
            self.dy2[q] = 1.0
        self.x[q] = (p.mean + 1).bfloat16()                     # x - mean = 1
        if s is not None:
            self.x2[q] = (s.mean + 1).bfloat16()
        if self.mask is not None:
            self.mask[q] = 255
        if self.rounding:
            q = torch.tensor(self.rounding, device=dev)
            big = torch.tensor([256.0, 258.0, 260.0, 516.0, 1032.0, 2064.0, 4096.0, -258.0, -1032.0, -4080.0],
                               device=dev)
            small = torch.tensor([0.25, 0.5, 1.0, -0.25, -0.5, -1.0], device=dev)
            shape = (len(self.rounding), C)
            self.dy[q] = big[torch.randint(0, len(big), shape, device=dev, generator=g)].bfloat16()
            self.dy2[q] = small[torch.randint(0, len(small), shape, device=dev, generator=g)].bfloat16()
            sign = lambda: torch.randint(0, 2, shape, device=dev, generator=g) * 2 - 1
            self.x[q] = (p.mean + sign() / 8.0).bfloat16()
            self.x2[q] = (s.mean + sign() / 8.0).bfloat16()
            self.mask[q] = 255

    def y_ref(self, i, n):
        return _y_ref(self.x[i:i + n], self.p.ca, self.p.cb, None, 1)

    def on(self, i, n):
        """The reference ReLU mask of rows i .. i + n - 1 (None: no mask)."""
        if self.kind in ("x", "y"):
            return self.y_ref(i, n).float() > 0
        return None if self.mask is None else _bits(self.mask[i:i + n], self.C)

    def g_ref(self, i, n):
        d = self.dy[i:i + n].float()
        if self.dy2 is not None:
            d = (d + self.dy2[i:i + n].float()).bfloat16().float()
        on = self.on(i, n)
        return d if on is None else torch.where(on, d, torch.zeros_like(d))

    def forward(self):
        """moco_bn_fwd_train_given on the same x and statistics: its y and mask bits against the reference, then y is
        the backward's input in mode "y"."""
        if self.kind not in ("x", "y"):
            return
        L = _lib()
        L.check(L.load().moco_bn_fwd_train_given(self.x.data_ptr(), None, self.y.data_ptr(), self.ybits.data_ptr(),
                                                 self.M, self.C, 1, self.p.layer(), None, STATS_GIVEN, None, 0,
                                                 L.cur_stream()), "moco_bn_fwd_train_given")
        torch.cuda.synchronize()
        for i in range(0, self.M, _rows(self.C)):
            n = min(_rows(self.C), self.M - i)
            want = self.y_ref(i, n)
            _equal("y", self.y[i:i + n], want, i)
            _equal("mask", self.ybits[i:i + n], _pack(want.float() > 0), i)

    def launch(self, ws):
        L = _lib()
        lib = L.load()
        p, ptr = self.p, lambda t: None if t is None else t.data_ptr()
        if self.kind in BWD_KINDS:
            L.check(lib.moco_bn_bwd(self.dy.data_ptr(), self.x.data_ptr(), ptr(self.y if self.kind == "y" else None), self.M,
                                    self.C, p.gamma.data_ptr(), p.beta.data_ptr(), p.mean.data_ptr(),
                                    p.invstd.data_ptr(), int(self.kind in ("x", "y")),
                                    int(self.kind in ("y", "none_res")), self.dx.data_ptr(), ptr(self.dres),
                                    self.dgamma.data_ptr(), self.dbeta.data_ptr(), ws.data_ptr(), ws.numel(),
                                    L.cur_stream()), "moco_bn_bwd")
            return
        bn = p.layer(self.dgamma, self.dbeta)
        sc = self.sc.layer(self.sc_dgamma, self.sc_dbeta) if self.sc is not None else None
        if self.dy2 is not None:
            L.check(lib.moco_bn_add_relu_bwd2(self.dy.data_ptr(), self.dy2.data_ptr(), self.x.data_ptr(),
                                              ptr(self.x2), self.mask.data_ptr(), self.M, self.C, bn, sc,
                                              self.dx.data_ptr(), ptr(self.dres), ws.data_ptr(), ws.numel(),
                                              L.cur_stream()), "moco_bn_add_relu_bwd2")
        else:
            L.check(lib.moco_bn_add_relu_bwd(self.dy.data_ptr(), self.x.data_ptr(), ptr(self.x2),
                                             self.mask.data_ptr(), self.M, self.C, bn, sc, self.dx.data_ptr(),
                                             ptr(self.dres), ws.data_ptr(), ws.numel(), L.cur_stream()),
                    "moco_bn_add_relu_bwd")

    def run(self, ws=None):
        self.forward()
        self.launch(ws if ws is not None else _ws(self.x.device))
        torch.cuda.synchronize()
        self.check()

    def check(self):
        """The sums from the exact reference g chunk by chunk (dresidual = g checked on the way), then dx and the
        shortcut's input gradient from the coefficients of the sums returned."""
        M, C, dev, p, s = self.M, self.C, self.x.device, self.p, self.sc
        S = torch.zeros(3, C, dtype=torch.float64, device=dev)
        B = torch.zeros(3, self.R, C, dtype=torch.float64, device=dev)
        for i in range(0, M, _rows(C)):
            n = min(_rows(C), M - i)
            ge = self.g_ref(i, n)
            if self.dres is not None and s is None:
                _equal("dresidual", self.dres[i:i + n].float(), ge, i)
            t = [ge.double(), ge.double() * (self.x[i:i + n].double() - p.mean.double())]
            if s is not None:
                t.append(ge.double() * (self.x2[i:i + n].double() - s.mean.double()))
            cta = torch.arange(i, i + n, device=dev) // self.L
            for k, (v, unit) in enumerate(zip(t, (4, 32, 32))):
                S[k] += v.sum(0)
                B[k].index_add_(0, cta, v.abs() * unit)
        assert float(B.max()) < 2 ** 24, "a CTA's fp32 partial could round"
        want_db = S[0].float()
        want_dg = (S[1] * p.invstd.double()).float()
        _assert_equal("dbeta", self.dbeta, want_db.cpu().numpy())
        _assert_equal("dgamma", self.dgamma, want_dg.cpu().numpy())
        if s is not None:
            _assert_equal("shortcut dbeta", self.sc_dbeta, want_db.cpu().numpy())
            _assert_equal("shortcut dgamma", self.sc_dgamma, (S[2] * s.invstd.double()).float().cpu().numpy())
        if M > 1 and self.planted:
            on = self.on(0, 1)                       # row 0 is planted: the planted rows' mask
            on = torch.ones(C, dtype=torch.bool, device=dev) if on is None else on[0]
            if self.kind in ("x", "y"):
                assert int(on.sum()) == C - 3 and not bool(on[[UNDERFLOW, ZEROS, TIE]].any())
            for sign in (-1, 1):                     # one planted row (g = 2, x - mean = 1) lost or repeated
                moved = ((S[0] + 2 * sign).float() != want_db) | (((S[1] + 2 * sign) * p.invstd.double()).float()
                                                                   != want_dg)
                assert bool(moved[on].all()), ("a planted row would go unseen", sign)
        coefs = [torch.from_numpy(v).to(dev) for v in _bwd_coefs(p.gamma.tolist(), p.mean.tolist(),
                                                                  p.invstd.tolist(), self.dbeta.tolist(),
                                                                  self.dgamma.tolist(), M)]
        if s is not None:
            coefs += [torch.from_numpy(v).to(dev) for v in _bwd_coefs(s.gamma.tolist(), s.mean.tolist(),
                                                                       s.invstd.tolist(), self.dbeta.tolist(),
                                                                       self.sc_dgamma.tolist(), M)]
        for i in range(0, M, _rows(C)):
            n = min(_rows(C), M - i)
            ge = self.g_ref(i, n)
            _equal("dx", self.dx[i:i + n], _fma32(coefs[0], ge, _fma32(coefs[1], self.x[i:i + n].float(),
                                                                        coefs[2])).bfloat16(), i)
            if s is not None:
                _equal("dresidual", self.dres[i:i + n], _fma32(coefs[3], ge, _fma32(
                    coefs[4], self.x2[i:i + n].float(), coefs[5])).bfloat16(), i)


# ---- 1. moco_bn_bwd, every mask mode

def _bwd_cases():
    out = []
    for a, M in enumerate(SMALL_M):
        for b, C in enumerate(CS):
            out.append((M, C, BWD_KINDS[(a + b) % 4]))
    for b, C in enumerate(CS):
        out += [(M, C, BWD_KINDS[(k + b) % 4]) for k, M in enumerate(_r_edges(C))]
    out += [(M, C, BWD_KINDS[k % 4]) for k, (C, M) in enumerate(_trip_edges(TRIP_BWD))]
    out += [(M, C, "x") for M, C in BN_SHAPES]       # the stem's, bn1's and bn2's backward at batch 256
    return out


@gpu
@pytest.mark.usefixtures("memory")
@pytest.mark.parametrize("M,C,kind", _bwd_cases())
def test_bn_bwd_exact(M, C, kind):
    """dbeta, dgamma, dx and dresidual of moco_bn_bwd exactly the reference's; with relu, its mask is the y > 0 of
    the forward's stored output (moco_bn_fwd_train_given, checked on the same x)."""
    _Bwd(M, C, kind, seed=M * 5 + C + BWD_KINDS.index(kind)).run()


# ---- 2. the downsample block's backward

def _sc_cases():
    out = []
    for a, M in enumerate(SMALL_M):
        for b, C in enumerate(CS):
            out.append((M, C, SC_KINDS[(a + b) % 3]))
    for b, C in enumerate(CS):
        out += [(M, C, SC_KINDS[(k + b) % 3]) for k, M in enumerate(_r_edges(C))]
    out += [(M, C, SC_KINDS[k % 2]) for k, (C, M) in enumerate(_trip_edges(TRIP_SC))]
    out += [(M, C, "sc2") for M, C in RESIDUAL_BN]   # ResNet-50's downsample bn3 / shortcut BN at batch 256
    out += [(200704, 512, "sc"), (12544, 2048, "bits")]
    return out


@gpu
@pytest.mark.usefixtures("memory")
@pytest.mark.parametrize("M,C,kind", _sc_cases())
def test_bn_add_relu_bwd_shortcut_exact(M, C, kind):
    """Both BatchNorms' dbeta and dgamma, dx and the shortcut's input gradient of moco_bn_add_relu_bwd(2) exactly the
    reference's; without the shortcut BN dresidual = g."""
    _Bwd(M, C, kind, seed=M * 3 + C + SC_KINDS.index(kind)).run()


# ---- 3. the apply without a residual, and the stem

FWD_MODES = [(relu, res, mask) for relu in (1, 0) for res in (False, True) for mask in (True, False)]


class _Fwd:
    """One forward case on cuda:0: moco_bn_fwd_train_given with the statistics given, or (train) moco_bn_fwd_train
    computing its own."""

    def __init__(self, M, C, relu, res, mask, seed, train=False):
        dev = torch.device("cuda:0")
        self.M, self.C, self.relu, self.train = M, C, relu, train
        g = torch.Generator(device=dev).manual_seed(seed)
        self.p = _Params(C, g, dev)
        self.x = torch.empty(M, C, dtype=torch.bfloat16, device=dev)
        self.r = torch.empty_like(self.x) if res else None
        for i in range(0, M, _rows(C)):
            n = min(_rows(C), M - i)
            self.x[i:i + n] = self.p.mean + torch.randint(-64, 65, (n, C), device=dev, generator=g,
                                                          dtype=torch.int8) / 8.0
            if res:
                self.r[i:i + n] = torch.randn(n, C, device=dev, generator=g) * 2
        if res:
            self.r[::7, ::3] = -0.0
        self.y = torch.empty_like(self.x)
        self.mask = torch.empty(M, C // 8, dtype=torch.uint8, device=dev) if mask else None
        self.stats = _running(C, dev, g) if train else None

    def run(self):
        L = _lib()
        lib = L.load()
        p, ptr = self.p, lambda t: None if t is None else t.data_ptr()
        if self.train:                               # the call's own statistics replace the given ones
            p.mean, p.invstd = torch.empty_like(p.mean), torch.empty_like(p.invstd)
            ws = _ws(self.x.device)
            L.check(lib.moco_bn_fwd_train(self.x.data_ptr(), ptr(self.r), self.y.data_ptr(), self.M, self.C,
                                          p.gamma.data_ptr(), p.beta.data_ptr(), self.stats[0].data_ptr(),
                                          self.stats[1].data_ptr(), self.stats[2].data_ptr(), 0.1, 1e-5, self.relu,
                                          p.mean.data_ptr(), p.invstd.data_ptr(), ws.data_ptr(), ws.numel(),
                                          L.cur_stream()), "moco_bn_fwd_train")
            torch.cuda.synchronize()
            p.ca, p.cb = _Bn.coefs(p)
        else:
            L.check(lib.moco_bn_fwd_train_given(self.x.data_ptr(), ptr(self.r), self.y.data_ptr(), ptr(self.mask),
                                                self.M, self.C, self.relu, p.layer(), None, STATS_GIVEN, None, 0,
                                                L.cur_stream()), "moco_bn_fwd_train_given")
        torch.cuda.synchronize()
        for i in range(0, self.M, _rows(self.C)):
            n = min(_rows(self.C), self.M - i)
            want = _y_ref(self.x[i:i + n], p.ca, p.cb, None if self.r is None else self.r[i:i + n], self.relu)
            _equal("y", self.y[i:i + n], want, i)
            if self.mask is not None:
                _equal("mask", self.mask[i:i + n], _pack(want.float() > 0), i)


def _fwd_cases():
    out = []
    for a, M in enumerate(SMALL_M):
        for b, C in enumerate(CS):
            out.append((M, C) + FWD_MODES[(a + 3 * b) % len(FWD_MODES)])
    out += [(M, C) + FWD_MODES[k % len(FWD_MODES)] for k, (C, M) in enumerate(_trip_edges(TRIP_FWD))]
    return out


@gpu
@pytest.mark.usefixtures("memory")
@pytest.mark.parametrize("M,C,relu,res,mask", _fwd_cases())
def test_bn_fwd_given_exact(M, C, relu, res, mask):
    """y and the mask bits of moco_bn_fwd_train_given (relu or not, no residual or an identity one) exactly the
    reference's."""
    _Fwd(M, C, relu, res, mask, seed=M * 7 + C + relu + 2 * res + 4 * mask).run()


@gpu
@pytest.mark.usefixtures("memory")
@pytest.mark.parametrize("M,C", BN_SHAPES)
def test_bn_fwd_train_output_exact(M, C):
    """moco_bn_fwd_train's y (relu, no residual: bn1, bn2 and the stem at batch 256) exactly the reference's with the
    call's own save_mean and save_invstd (their exact test is the conv1x1 envelope's)."""
    _Fwd(M, C, 1, False, False, seed=M + C, train=True).run()


# (N, H, W, C): the stem at batch 256, odd and even H and W down to 1, C up to the pool's 2048-channel table
STEM_SHAPES = [(256, 112, 112, 64), (3, 1, 1, 64), (2, 1, 2, 128), (2, 2, 1, 256), (3, 2, 2, 64), (2, 7, 5, 512),
               (2, 6, 9, 64), (1, 3, 4, 1024), (2, 5, 6, 2048), (4, 11, 8, 64)]


@gpu
@pytest.mark.usefixtures("memory")
@pytest.mark.parametrize("N,H,W,C", STEM_SHAPES)
def test_stem_bn_relu_maxpool_and_backward_exact(N, H, W, C):
    """moco_bn_relu_maxpool_fwd_train's y and tap bytes exactly _pool_reference of the exact BatchNorm + ReLU (the
    call's own statistics); then moco_maxpool3x3s2_bwd's g exactly _pool_bwd_reference and moco_bn_bwd (relu, mask
    from x) on it exactly the reference's."""
    L = _lib()
    lib = L.load()
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(N * 100 + H * 7 + W + C)
    M, OH, OW = N * H * W, (H - 1) // 2 + 1, (W - 1) // 2 + 1
    p = _Params(C, g, dev)
    x = torch.empty(N, H, W, C, dtype=torch.bfloat16, device=dev)
    imgs = max(1, 2 ** 22 // (H * W * C))
    for n0 in range(0, N, imgs):
        k = min(imgs, N - n0)
        x[n0:n0 + k] = torch.randint(-3, 4, (k, H, W, C), device=dev, generator=g, dtype=torch.int8) * 0.5
    fwd = types.SimpleNamespace(gamma=p.gamma, beta=p.beta, mean=torch.empty(C, device=dev),
                                invstd=torch.empty(C, device=dev))
    y = torch.empty(N, OH, OW, C, dtype=torch.bfloat16, device=dev)
    taps = torch.empty(N, OH, OW, C, dtype=torch.uint8, device=dev)
    ws = _ws(dev)
    from moco_b200.bn import _layer
    L.check(lib.moco_bn_relu_maxpool_fwd_train(
        x.data_ptr(), y.data_ptr(), taps.data_ptr(), N, H, W, C,
        _layer(p.gamma, p.beta, fwd.mean, fwd.invstd, _running(C, dev, g) + (0.1, 1e-5)), ws.data_ptr(), ws.numel(),
        L.cur_stream()), "moco_bn_relu_maxpool_fwd_train")
    torch.cuda.synchronize()
    ca, cb = _Bn.coefs(fwd)
    nchw = lambda t: t.permute(0, 3, 1, 2)
    rows = lambda t: t.permute(0, 2, 3, 1).reshape(-1, C)
    for n0 in range(0, N, imgs):
        k = min(imgs, N - n0)
        v = _y_ref(x[n0:n0 + k].reshape(-1, C), ca, cb, None, 1).view(k, H, W, C)
        m, tap = _pool_reference(nchw(v))
        _equal("y", y[n0:n0 + k].reshape(-1, C).float(), rows(m), n0 * OH * OW)
        _equal("taps", taps[n0:n0 + k].reshape(-1, C), rows(tap), n0 * OH * OW)
    dyp = torch.randint(-8, 9, (N, OH, OW, C), device=dev, generator=g, dtype=torch.int8).bfloat16() / 4
    gi = torch.empty_like(x)
    L.check(lib.moco_maxpool3x3s2_bwd(dyp.data_ptr(), taps.data_ptr(), gi.data_ptr(), N, H, W, C, L.cur_stream()),
            "moco_maxpool3x3s2_bwd")
    torch.cuda.synchronize()
    for n0 in range(0, N, imgs):
        k = min(imgs, N - n0)
        want = _pool_bwd_reference(nchw(dyp[n0:n0 + k]), nchw(taps[n0:n0 + k]), H, W)
        _equal("g", gi[n0:n0 + k].reshape(-1, C), rows(want), n0 * H * W)
    del y, dyp
    _Bwd(M, C, "x", 0, given=(p, gi.view(M, C), x.view(M, C))).run(ws)


# ---- 4. one workspace, and CUDA graphs

@gpu
@pytest.mark.usefixtures("memory")
def test_one_workspace_in_turn():
    """moco_bn_bwd at C = 64 (1 slab, 264 CTAs), the shortcut backward at C = 2048 (32 slabs, 3 sums), then
    moco_bn_bwd at C = 64 again on one workspace zeroed once: each call matches its own reference, so each re-arms
    the slab counters the next one uses."""
    ws = _ws(torch.device("cuda:0"))
    _Bwd(50176, 64, "x", 61).run(ws)
    _Bwd(12544, 2048, "sc2", 62).run(ws)
    _Bwd(50177, 64, "x", 63).run(ws)


@gpu
@pytest.mark.usefixtures("memory")
def test_both_backwards_graph_replay():
    """moco_bn_bwd (mask from x) and the shortcut backward captured in one CUDA graph and replayed twice on inputs
    refreshed in place: exact each time."""
    a, b = _Bwd(20000, 256, "x", 71), _Bwd(12544, 512, "sc2", 72)
    ws = _ws(a.x.device)
    a.run(ws)
    b.run(ws)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        a.launch(ws)
        b.launch(ws)
    for _ in range(2):
        a.fill()
        b.fill()
        a.forward()
        graph.replay()
        torch.cuda.synchronize()
        a.check()
        b.check()


# ---- the reference helpers, by hand (no GPU)

def test_apply_grid_and_trip_edges_by_hand():
    """_apply_grid on cases computed by hand, and the trip edges' M straddle one or two whole trips."""
    assert _apply_grid(1, 8, 2) == 1 and _apply_grid(2048, 8, 2) == 1 and _apply_grid(2049, 8, 2) == 2
    assert _apply_grid(TRIP_FWD, 8, 2) == 264 and _apply_grid(TRIP_FWD - 2048, 8, 2) == 263
    assert _apply_grid(10 ** 9, 2, 3) == 396 and _apply_grid(TRIP_SC + 1, 2, 2) == 264
    for trip, unroll, ctas in ((TRIP_FWD, 8, 2), (TRIP_BWD, 2, 3), (TRIP_SC, 2, 2)):
        edges = _trip_edges(trip)
        assert len(edges) == 9
        for j in range(0, 9, 3):
            (C, M0), k = edges[j], (1, 1, 2)[j // 3]
            trips = []
            for _, M in edges[j:j + 3]:
                V = M * C // 8
                trips.append(-(-V // (_apply_grid(V, unroll, ctas) * 256 * unroll)))
            assert trips == [k, k, k + 1], (trip, C, trips)
    assert _trip_edges(TRIP_BWD)[:3] == [(64, 25343), (64, 25344), (64, 25345)]
    # 32 slabs, R <= 8: 29 passes give R = 8 (4 each), 33 passes 8 passes each, R = 5
    assert _r_edges(2048) == [896, 897, 898, 1024, 1025, 1026]


def test_underflow_channel_by_hand():
    """gamma = 1e-42, beta = 0: every z = fmaf(x, ca, cb) over the inputs' range is a subnormal below 2^-134, so bf16
    stores zero and the ReLU mask is off, though z > 0 in half of the rows; ca = 2^-136, beta = 0: z = (x - mean)
    2^-136 is on exactly above the tie at x - mean = 4; the other channels' planted rows (x - mean = 1) have their
    mask on, channel 2's (beta = -1e4) off."""
    g = torch.Generator().manual_seed(5)
    p = _Params(256, g, torch.device("cpu"))
    d = torch.arange(-64, 65, dtype=torch.float32).unsqueeze(1) / 8.0
    x = (p.mean + d).bfloat16()
    assert torch.equal(x.float(), p.mean + d)                   # the 1/8 grid is exact in bf16
    z = _fma32(x.float(), p.ca, p.cb)[:, UNDERFLOW]
    assert bool((z > 0).any()) and float(z.abs().max()) < 2.0 ** -134
    y = _y_ref(x, p.ca, p.cb, None, 1)
    assert not bool((y[:, UNDERFLOW].float() != 0).any())
    assert torch.equal(_fma32(x.float(), p.ca, p.cb)[:, TIE], d[:, 0] * 2.0 ** -136)
    assert torch.equal(y[:, TIE].float() > 0, d[:, 0] > 4)
    on = _y_ref((p.mean + 1).bfloat16().unsqueeze(0), p.ca, p.cb, None, 1)[0].float() > 0
    assert int(on.sum()) == 253 and not bool(on[[UNDERFLOW, ZEROS, TIE]].any())
    # bf16's smallest subnormal is 2^-133: 2^-134 is a tie to even (zero), just above it rounds up
    t = torch.tensor([2.0 ** -134, 2.0 ** -134 + 2.0 ** -149, 2.0 ** -133]).bfloat16().float().tolist()
    assert t == [0.0, 2.0 ** -133, 2.0 ** -133]
