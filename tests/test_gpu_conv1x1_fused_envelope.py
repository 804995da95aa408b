"""The two fused 1x1-convolution kernels that carry BatchNorm work in their epilogues (csrc/conv1x1_sm90.cu) over the
whole envelope include/moco_b200.h promises, against exact references that share no code with them:
moco_conv1x1_dgrad_bn_bwd followed by moco_bn_bwd_apply_given, and moco_conv1x1_bn_add_relu_fwd; and
moco_bn_add_relu_bwd2, the other caller of the same backward code, at ResNet-50's batch-256 residual BatchNorm shapes.
Every output is compared exactly (torch.equal / np.array_equal on values: the sign of an exact zero from the wgmma
accumulator is not part of the contract).

Backward inputs.  w [K, C] is +1 in row 0 and s_c = +-1 in row j_c (j covers every 64-row K chunk and row K - 1), dh is
in {-1, -1/2, 0, 1/2, 1}, so dX = dh . w is exact in any order, in float64 and in the kernel's fp32 accumulator.  dy2
is on a 1/4 grid, x and mean on a common 1/8 grid (the kernel's fp32 x - mean is exact), gamma and invstd arbitrary.
x - mean is in [-8, 8] with the sign of dX + dy2, so that at the large M S2 outgrows fp32's 24 bits (only the fp64
finish and bn_bwd_channel's double product keep it) while each CTA's partials stay exact.
A few rounding rows carry |dX| in 257 .. 4083 (exact bf16 ties included) and x - mean = +-1/8.  The reference is
    g = mask . bf16(fp32(bf16(dX) + dy2)),   dbeta = fp32(S1),   dgamma = fp32(fp64(S2 * invstd))
with S1 = sum g and S2 = sum g (x - mean) taken exactly in float64; that every fp32 partial the kernel forms is exact
is asserted from the data: in each CTA row chunk of bn_bwd_reduce_plan (_plan with unroll 4) and each channel, the sum
of |g| in units of 1/4 and of |g (x - mean)| in units of 1/32 stays below 2^24.  Planted rows (g = 2, x - mean = 1,
mask on) at the chunk and tile edges, the ragged last tile and row M - 1 must each move dbeta or dgamma in every
channel when dropped or repeated.  dx = bf16(fmaf(cA, g, fmaf(cB, x, cD))) with bwd_coefs (csrc/bn_nhwc.cu)
evaluated per channel: its products in numpy float32 in source order (cB = ((-k1) m2) is), inv_m = (float)(1.0 / M),
and its fmaf in Fraction; the per-element fmaf through _fma32 (float64 rounded to odd, then to float32).

Forward inputs.  With MOCO_BN_STATS_GIVEN, w in {-1, 0, 1} and x in {-4, -1, 0, 1, 4}, every fourth row
8 w[row % Cout] + u with u in {-1, 0, 1}: h = x . w^T is exact, reaches hundreds and its bf16 rounding hits ties; the
statistics, gamma and beta are arbitrary floats and r is random bf16 with some -0.  Without it, the statistics
envelope's design (h an integer in [-2, 2], shift row 0, planted rows) and its _channel_stats check the statistics the
call computes; the shortcut BN's statistics, when not given, are checked the same way on r in {-2, .., 2}.  y is then
    ca = gamma * invstd,  cb = fmaf(-mean, ca, beta),  y = bf16(max(fp32(fmaf(bf16(h), ca, cb) + r), 0))
with r = bf16(fp32(fmaf(s, ca2, cb2) + 0)) through a shortcut BN, and the mask bits are y > 0, 8 per byte.

Contractions.  cuobjdump -sass of the library nvcc 12.9 builds (-O3, default -fmad=true) shows only the source's
explicit fmaf: bn_bwd_apply_kernel<2, 3, false, false> (what moco_bn_bwd_apply_given runs) has 48 FMUL and 64 FFMA,
i.e. per channel bwd_coefs' 6 multiplies and 2 fmaf and per element the 2 fmaf of dx and 1 of the mask test; each
conv1x1_bn_apply_kernel has 1 FMUL, 1 FFMA per coefficient thread and 1 FFMA, 1 FADD and 1 FMNMX per element (twice
that with the shortcut BN); conv1x1_dgrad_bn_bwd_kernel's bn_bwd_channel is one DMUL per slab.

Size.  dh of the K = 4096 case is 4.3 GB (TMA reads of the A operand past 2^32 bytes) and the Cout = 2048 forward at
M = 1,048,705 has r and y of 4.3 GB each.  An [M, C] backward tensor past 2^32 bytes would need three 4.3 GB tensors
(x, dy2, g) and is left out; the kernel reaches x, dy2, the mask and g only through TMA maps, addressed as dh is.
Every case stays under 10 GB of device memory (asserted)."""
import gc
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

from tests.test_gpu_conv1x1_envelope import (_Case, _assert_equal, _check_stats, _f32, _fill_x, _new_ws, _plan,
                                              _planted, _q, _r_changes, _round, _running, _totals, _weights)

gpu = pytest.mark.gpu
MEM_LIMIT = 10 * 10 ** 9
STATS_GIVEN, SC_STATS_GIVEN = 1, 2           # MOCO_BN_STATS_GIVEN, MOCO_BN_SC_STATS_GIVEN


@pytest.fixture
def memory():
    """Each GPU case under MEM_LIMIT bytes of device memory; its tensors freed afterwards.  The traceback of a failed
    case (kept in sys.last_traceback for a debugger) holds its tensors: it is dropped first, so that one large failing
    case does not push the next one over the limit."""
    sys.last_type = sys.last_value = sys.last_traceback = sys.last_exc = None
    gc.collect()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    yield
    peak = torch.cuda.max_memory_allocated() - base
    print(f"\npeak device memory {peak / 1e9:.2f} GB")
    torch.cuda.empty_cache()
    assert peak <= MEM_LIMIT, peak


# ---- exact arithmetic helpers

def _fma32(a, b, c):
    """fmaf(a, b, c) on float32 tensors (broadcast), correctly rounded.  In float64 a * b is exact; p + c is rounded
    to odd (its TwoSum error e != 0 and an even last significand bit: one ulp toward e), and rounding that to float32's
    24 bits is then the single rounding of the exact value (53 >= 24 + 2)."""
    a, b, c = torch.broadcast_tensors(a.double(), b.double(), c.double())
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    inf = torch.full_like(s, float("inf"))
    odd = torch.where(e > 0, inf, -inf)
    fix = (e != 0) & ((s.view(torch.int64) & 1) == 0)
    return torch.where(fix, torch.nextafter(s, odd), s).float()


def _fmaf(a, b, c):
    """One fmaf on float32 scalars, exactly in Fraction."""
    return _f32(_q(a) * _q(b) + _q(c))


def _bits(mask, C):
    """uint8 [n, C / 8] -> bool [n, C], bit k of byte v is channel 8 v + k."""
    sh = torch.arange(8, device=mask.device, dtype=torch.uint8)
    return ((mask.unsqueeze(-1) >> sh) & 1).bool().view(mask.shape[0], C)


def _pack(on):
    """bool [n, C] -> uint8 [n, C / 8] (relu_bits' order)."""
    n, C = on.shape
    sh = torch.arange(8, device=on.device, dtype=torch.uint8)
    return (on.view(n, C // 8, 8).to(torch.uint8) << sh).sum(-1).to(torch.uint8)


def _rows(C):
    """Row chunk of the references: 2^22 elements (32 MB per float64 temporary)."""
    return max(1, 2 ** 22 // C)


def _equal(name, got, want, i=0):
    if not torch.equal(got, want):
        bad = (got != want).nonzero()[0].tolist()
        raise AssertionError(f"{name}[{i + bad[0]}, {bad[1]}] = {float(got[tuple(bad)])}, exact "
                             f"{float(want[tuple(bad)])} ({int((got != want).sum())} elements differ in this chunk)")


def _lib():
    from moco_b200 import _lib as L
    return L


# ---- the backward: moco_conv1x1_dgrad_bn_bwd + moco_bn_bwd_apply_given

def _bwd_coefs(gamma, mean, invstd, dbeta, dgamma, M):
    """bwd_coefs (csrc/bn_nhwc.cu) per channel: (cA, cB, cD) as float32 arrays."""
    inv_m = np.float32(1.0 / M)
    out = np.empty((3, len(gamma)), dtype=np.float32)
    for c, (ga, mu, s, db, dg) in enumerate(zip(gamma, mean, invstd, dbeta, dgamma)):
        k1 = np.float32(ga) * np.float32(s)
        m1 = np.float32(db) * inv_m
        m2 = np.float32(dg) * inv_m
        cB = (-k1 * m2) * np.float32(s)
        out[:, c] = k1, cB, _fmaf(-cB, mu, -k1 * m1)
    return out


class _Dgrad:
    """One backward case on cuda:0: C the BatchNorm's channels (the convolution's Cin), K its Cout (the GEMM's K)."""

    def __init__(self, C, K, M, seed):
        dev = torch.device("cuda:0")
        self.C, self.K, self.M = C, K, M
        self.g = torch.Generator(device=dev).manual_seed(seed)
        j = (torch.arange(C, device=dev) % (K // 64)) * 64 + torch.randint(0, 64, (C,), device=dev, generator=self.g)
        self.j = j.clamp_min(1)
        self.j[-1] = K - 1
        self.s = (torch.randint(0, 2, (C,), device=dev, generator=self.g) * 2 - 1).float()
        w = torch.zeros(K, C, device=dev)
        w[0] = 1
        w[self.j, torch.arange(C, device=dev)] = self.s
        self.w = w.bfloat16()
        self.gamma = torch.randn(C, device=dev, generator=self.g)
        self.invstd = torch.rand(C, device=dev, generator=self.g) + 0.3
        self.mean = torch.randint(-8, 9, (C,), device=dev, generator=self.g) / 8.0
        self.dh = torch.empty(M, K, dtype=torch.bfloat16, device=dev)
        self.x = torch.empty(M, C, dtype=torch.bfloat16, device=dev)
        self.dy2 = torch.empty_like(self.x)
        self.mask = torch.empty(M, C // 8, dtype=torch.uint8, device=dev)
        _, per, self.R = _plan(M, C, 4)
        self.L = 32 * per                                      # rows per CTA chunk
        self.planted = sorted(set(_planted(M, C, 4)) | {0})
        cand = [M // 5, 2 * M // 5, M // 2 + 1, 3 * M // 5, 4 * M // 5, M - 2]
        self.rounding = sorted({r for r in cand if 0 <= r < M} - set(self.planted))
        self.fill()
        self.gout = torch.empty_like(self.x)
        self.dx = torch.empty_like(self.x)
        self.dgamma = torch.empty(C, device=dev)
        self.dbeta = torch.empty(C, device=dev)

    def fill(self):
        """New inputs in place (graph replays read the same buffers)."""
        M, C, K, g, dev = self.M, self.C, self.K, self.g, self.x.device
        step = max(1, 2 ** 26 // K)
        for i in range(0, M, step):
            n = min(step, M - i)
            self.dh[i:i + n] = torch.randint(-2, 3, (n, K), device=dev, generator=g, dtype=torch.int8) * 0.5
        for i in range(0, M, _rows(C)):
            n = min(_rows(C), M - i)
            self.dy2[i:i + n] = torch.randint(-8, 9, (n, C), device=dev, generator=g, dtype=torch.int8) * 0.25
            d = torch.randint(0, 65, (n, C), device=dev, generator=g, dtype=torch.int8) / 8.0
            self.x[i:i + n] = self.mean + d * torch.sign(self.dX(i, n) + self.dy2[i:i + n].float())
            self.mask[i:i + n] = torch.randint(0, 256, (n, C // 8), device=dev, generator=g, dtype=torch.uint8)
        p = torch.tensor(self.planted, device=dev)
        self.dh[p] = 0
        self.dh[p, 0] = 1                                      # dX = 1
        self.dy2[p] = 1                                        # g = 2
        self.x[p] = (self.mean + 1).bfloat16()                 # x - mean = 1
        self.mask[p] = 255
        if self.rounding:
            q = torch.tensor(self.rounding, device=dev)
            big = torch.tensor([260.0, 300.0, 516.0, 1032.0, 2064.0, 4080.0, -260.0, -1032.0], device=dev)
            vals = torch.tensor([-3.0, -1.5, -1.0, -0.5, 0.5, 1.0, 1.5, 3.0], device=dev)
            pick = torch.randint(0, 8, (len(self.rounding), K), device=dev, generator=g)
            self.dh[q] = vals[pick].bfloat16()
            self.dh[q, 0] = big[torch.arange(len(self.rounding), device=dev) % 8].bfloat16()   # |dX| in 257 .. 4083
            sgn = torch.randint(0, 2, (len(self.rounding), C), device=dev, generator=g) * 2 - 1
            self.x[q] = (self.mean + sgn / 8.0).bfloat16()
            self.mask[q] = 255

    def dX(self, i, n):
        """The exact dX of rows i .. i + n - 1 (float32)."""
        dh = self.dh[i:i + n]
        return dh[:, :1].float() + dh[:, self.j].float() * self.s

    def launch(self, ws):
        L = _lib()
        from moco_b200.bn import _layer
        lib = L.load()
        bn = _layer(self.gamma, None, self.mean, self.invstd, dgamma=self.dgamma, dbeta=self.dbeta)
        L.check(lib.moco_conv1x1_dgrad_bn_bwd(self.dh.data_ptr(), self.w.data_ptr(), self.gout.data_ptr(), self.M,
                                              self.C, self.K, self.x.data_ptr(), self.mask.data_ptr(),
                                              self.dy2.data_ptr(), None, bn, None, ws.data_ptr(), ws.numel(),
                                              L.cur_stream()), "moco_conv1x1_dgrad_bn_bwd")
        L.check(lib.moco_bn_bwd_apply_given(self.gout.data_ptr(), self.x.data_ptr(), None, self.M, self.C, bn, None,
                                            self.dx.data_ptr(), None, L.cur_stream()), "moco_bn_bwd_apply_given")

    def run(self, ws=None):
        self.launch(ws if ws is not None else _new_ws(self.x.device))
        torch.cuda.synchronize()
        self.check(self.gout, self.dbeta, self.dgamma, self.dx)

    def g_exact(self, i, n):
        dXb = self.dX(i, n).bfloat16().float()
        gs = (dXb + self.dy2[i:i + n].float()).bfloat16().float()
        return torch.where(_bits(self.mask[i:i + n], self.C), gs, torch.zeros_like(gs))

    def check(self, g, dbeta, dgamma, dx):
        """g against its reference row chunk by row chunk, then dbeta / dgamma from the exact sums, then dx."""
        M, C, dev = self.M, self.C, self.x.device
        s1 = torch.zeros(C, dtype=torch.float64, device=dev)
        s2 = torch.zeros_like(s1)
        b1 = torch.zeros(self.R, C, dtype=torch.float64, device=dev)
        b2 = torch.zeros_like(b1)
        for i in range(0, M, _rows(C)):
            n = min(_rows(C), M - i)
            ge = self.g_exact(i, n)
            _equal("g", g[i:i + n].float(), ge, i)
            t = ge.double() * (self.x[i:i + n].double() - self.mean.double())
            s1 += ge.double().sum(0)
            s2 += t.sum(0)
            cta = torch.arange(i, i + n, device=dev) // self.L
            b1.index_add_(0, cta, ge.double().abs() * 4)
            b2.index_add_(0, cta, t.abs() * 32)
        assert float(b1.max()) < 2 ** 24 and float(b2.max()) < 2 ** 24, "a CTA's fp32 partial could round"
        want_db = s1.float()
        want_dg = (s2 * self.invstd.double()).float()
        _assert_equal("dbeta", dbeta, want_db.cpu().numpy())
        _assert_equal("dgamma", dgamma, want_dg.cpu().numpy())
        if M > 1:
            for sign in (-1, 1):                     # one planted row (g = 2, x - mean = 1) lost or repeated
                moved = ((s1 + 2 * sign).float() != want_db) | (((s2 + 2 * sign) * self.invstd.double()).float()
                                                                != want_dg)
                assert bool(moved.all()), ("a planted row would go unseen", sign)
        coefs = _bwd_coefs(self.gamma.tolist(), self.mean.tolist(), self.invstd.tolist(), dbeta.tolist(),
                           dgamma.tolist(), M)
        cA, cB, cD = (torch.from_numpy(v).to(dev) for v in coefs)
        for i in range(0, M, _rows(C)):
            n = min(_rows(C), M - i)
            want = _fma32(cA, self.g_exact(i, n), _fma32(cB, self.x[i:i + n].float(), cD)).bfloat16()
            _equal("dx", dx[i:i + n], want, i)


D_CS = [128, 256, 512, 1024, 2048]
D_KS = [64, 192, 256, 320, 1088, 4096]          # 1, 3, 4, 5, 17 and 64 K chunks
D_SMALL_M = [1, 31, 127, 128, 129, 255, 256, 257]


def _dgrad_cases():
    out = []
    for a, M in enumerate(D_SMALL_M):
        for b, C in enumerate(D_CS):
            out.append((C, D_KS[(a + b) % len(D_KS)], M))
    for b, C in enumerate(D_CS):
        ch = _r_changes(C, 802816, 4)
        rs = [_plan(m, C, 4)[2] for m in ch]
        top = rs.index(max(rs))
        out += [(C, D_KS[(b + k) % 2], m + k) for m in ch[top:top + 2] for k in (-1, 0, 1) if m + k >= 1]
    out += [
        (256, 64, 802816), (256, 128, 802816), (512, 128, 200704), (512, 256, 200704),   # the batch-256 table
        (2048, 512, 12544),      # stage 4's identity-block conv1 at batch 256
        (2048, 512, 50176),      # 16 column slices, R = 8: about 49 tiles per CTA
        (128, 4096, 524545),     # dh is 4.3 GB: A-operand offsets past 2^32; 64 K chunks through a 2-stage ring
    ]
    return out


@gpu
@pytest.mark.usefixtures("memory")
@pytest.mark.parametrize("C,K,M", _dgrad_cases())
def test_dgrad_bn_bwd_exact(C, K, M):
    """g, dbeta, dgamma and dx of moco_conv1x1_dgrad_bn_bwd + moco_bn_bwd_apply_given exactly the reference's."""
    _Dgrad(C, K, M, seed=M * 5 + K * 3 + C).run()


# ResNet-50's residual BatchNorms of the identity blocks at batch 256 (M, C)
RESIDUAL_BN = [(802816, 256), (200704, 512), (50176, 1024), (12544, 2048)]


@gpu
@pytest.mark.usefixtures("memory")
@pytest.mark.parametrize("M,C", RESIDUAL_BN)
def test_bn_add_relu_bwd2_exact(M, C):
    """moco_bn_add_relu_bwd2 with dy = the exact bf16(dX) and dy2: its dres is g, and dres, dbeta, dgamma and dx are
    exactly the dgrad references."""
    L = _lib()
    from moco_b200.bn import _layer
    lib = L.load()
    case = _Dgrad(C, 64, M, seed=M + C)
    dy = torch.empty_like(case.x)
    for i in range(0, M, _rows(C)):
        n = min(_rows(C), M - i)
        dy[i:i + n] = case.dX(i, n).bfloat16()
    case.dh = None
    ws = torch.zeros(lib.moco_bn_workspace_bytes(), dtype=torch.uint8, device=dy.device)
    bn = _layer(case.gamma, None, case.mean, case.invstd, dgamma=case.dgamma, dbeta=case.dbeta)
    L.check(lib.moco_bn_add_relu_bwd2(dy.data_ptr(), case.dy2.data_ptr(), case.x.data_ptr(), None,
                                      case.mask.data_ptr(), M, C, bn, None, case.dx.data_ptr(), case.gout.data_ptr(),
                                      ws.data_ptr(), ws.numel(), L.cur_stream()), "moco_bn_add_relu_bwd2")
    torch.cuda.synchronize()
    case.dX = lambda i, n: dy[i:i + n].float()
    case.check(case.gout, case.dbeta, case.dgamma, case.dx)


# ---- the forward: moco_conv1x1_bn_add_relu_fwd

class _Bn:
    """One BatchNorm's parameters, statistics and running statistics."""

    def __init__(self, C, g, dev, given):
        self.gamma = torch.rand(C, device=dev, generator=g) + 0.5
        self.beta = torch.randn(C, device=dev, generator=g)
        if given:                                    # arbitrary floats (h reaches hundreds)
            self.mean = torch.randn(C, device=dev, generator=g) * 8
            self.invstd = (torch.rand(C, device=dev, generator=g) + 0.5) / 32
        else:
            self.mean, self.invstd = torch.empty(C, device=dev), torch.empty(C, device=dev)
        self.stats = _running(C, dev, g)

    def layer(self, momentum=0.1, eps=1e-5):
        from moco_b200.bn import _layer
        return _layer(self.gamma, self.beta, self.mean, self.invstd, self.stats + (momentum, eps))

    def snapshot(self):
        return [t.clone() for t in (self.mean, self.invstd) + self.stats]

    def unchanged(self, before):
        for u, v in zip(before, [self.mean, self.invstd] + list(self.stats)):
            assert torch.equal(u, v)

    def coefs(self):
        """bn_apply_kernel's ca = gamma * invstd, cb = fmaf(-mean, ca, beta) (float32 tensors)."""
        ca = self.gamma.cpu().numpy() * self.invstd.cpu().numpy()
        cb = [_fmaf(-m, a, b) for m, a, b in zip(self.mean.tolist(), ca, self.beta.tolist())]
        dev = self.gamma.device
        return torch.from_numpy(ca).to(dev), torch.tensor(np.array(cb, dtype=np.float32), device=dev)


class _Apply:
    """One forward case on cuda:0: y = relu(bn(x . w^T) + r) (r through a shortcut BN with `shortcut`)."""

    def __init__(self, Cin, Cout, M, seed, shortcut, given, mask=True):
        dev = torch.device("cuda:0")
        self.Cin, self.Cout, self.M, self.shortcut, self.given = Cin, Cout, M, shortcut, given
        self.g = g = torch.Generator(device=dev).manual_seed(seed)
        self.bn = _Bn(Cout, g, dev, given & STATS_GIVEN)
        self.sc = _Bn(Cout, g, dev, given & SC_STATS_GIVEN) if shortcut else None
        self.planted = _planted(M, Cout)
        self.x = torch.empty(M, Cin, dtype=torch.bfloat16, device=dev)
        if given & STATS_GIVEN:
            self.w = torch.randint(-1, 2, (Cout, Cin), device=dev, generator=g).bfloat16()
        else:
            self.w, self.j, self.s = _weights(Cin, Cout, g)
        self.fill_x()
        self.r = torch.empty(M, Cout, dtype=torch.bfloat16, device=dev)
        if shortcut and not given & SC_STATS_GIVEN:    # the shortcut BN's statistics are computed: r in {-2, .., 2}
            for i in range(0, M, _rows(Cout)):
                n = min(_rows(Cout), M - i)
                self.r[i:i + n] = torch.randint(-2, 3, (n, Cout), device=dev, generator=g, dtype=torch.int8)
            self.r[0] = -2
            if self.planted:
                self.r[torch.tensor(self.planted, device=dev)] = 2
        else:
            for i in range(0, M, _rows(Cout)):
                n = min(_rows(Cout), M - i)
                self.r[i:i + n] = torch.randn(n, Cout, device=dev, generator=g) * 2
            self.r[::7, ::3] = -0.0
        self.y = torch.empty_like(self.r)
        self.mask = torch.empty(M, Cout // 8, dtype=torch.uint8, device=dev) if mask else None

    def fill_x(self):
        M, Cin, dev, g = self.M, self.Cin, self.x.device, self.g
        if not self.given & STATS_GIVEN:
            _fill_x(self.x, g, self.planted)
            return
        vals = torch.tensor([-4.0, -1.0, 0.0, 1.0, 4.0], device=dev)
        step = max(1, 2 ** 24 // Cin)
        for i in range(0, M, step):
            n = min(step, M - i)
            self.x[i:i + n] = vals[torch.randint(0, 5, (n, Cin), device=dev, generator=g)].bfloat16()
            rows = torch.arange(i + (1 - i) % 4, i + n, 4, device=dev)          # rows = 1 mod 4: 8 w[row % Cout] + u
            u = torch.randint(-1, 2, (len(rows), Cin), device=dev, generator=g)
            self.x[rows] = (self.w[rows % self.Cout] * 8 + u).bfloat16()

    def h(self, i, n):
        """The exact h = x . w^T of rows i .. i + n - 1 (float32)."""
        xc = self.x[i:i + n]
        if self.given & STATS_GIVEN:
            return (xc.double() @ self.w.double().t()).float()
        return xc[:, :1].float() + xc[:, self.j].float() * self.s

    def launch(self, ws, momentum=0.1, eps=1e-5):
        L = _lib()
        lib = L.load()
        L.check(lib.moco_conv1x1_bn_add_relu_fwd(
            self.x.data_ptr(), self.w.data_ptr(), self.r.data_ptr(), self.y.data_ptr(),
            None if self.mask is None else self.mask.data_ptr(), self.M, self.Cin, self.Cout,
            self.bn.layer(momentum, eps), self.sc.layer(momentum, eps) if self.sc else None, self.given,
            ws.data_ptr(), ws.numel(), L.cur_stream()), "moco_conv1x1_bn_add_relu_fwd")

    def run(self, ws=None, momentum=0.1, eps=1e-5):
        L = _lib()
        lib = L.load()
        if ws is None:
            ws = torch.zeros(max(lib.moco_conv1x1_workspace_bytes(), lib.moco_bn_workspace_bytes()),
                             dtype=torch.uint8, device=self.x.device)
        before = self.snapshots()
        self.launch(ws, momentum, eps)
        torch.cuda.synchronize()
        self.check(before, momentum, eps)

    def snapshots(self):
        return self.bn.snapshot(), self.sc.snapshot() if self.sc else None

    def check(self, before, momentum, eps):
        """The statistics the call computed (or left alone), then y and the mask bits, chunk by chunk."""
        M, C, dev = self.M, self.Cout, self.x.device
        if self.given & STATS_GIVEN:
            self.bn.unchanged(before[0])
        else:
            h = torch.empty(M, C, dtype=torch.bfloat16, device=dev)
            for i in range(0, M, _rows(C)):
                n = min(_rows(C), M - i)
                h[i:i + n] = self.h(i, n)
            _check_stats(_totals(h), M, C, momentum, eps, before[0][2:], self.bn.stats, self.bn.mean,
                         self.bn.invstd, 2)
            del h
        if self.sc is not None:
            if self.given & SC_STATS_GIVEN:
                self.sc.unchanged(before[1])
            else:
                _check_stats(_totals(self.r), M, C, momentum, eps, before[1][2:], self.sc.stats, self.sc.mean,
                             self.sc.invstd, 4)
        ca, cb = self.bn.coefs()
        ca2, cb2 = self.sc.coefs() if self.sc else (None, None)
        for i in range(0, M, _rows(C)):
            n = min(_rows(C), M - i)
            r = self.r[i:i + n].float()
            if self.sc is not None:
                r = (_fma32(r, ca2, cb2) + 0.0).bfloat16().float()
            t = _fma32(self.h(i, n).bfloat16().float(), ca, cb)
            z = t + r
            want = torch.maximum(z, torch.zeros_like(z)).bfloat16()
            _equal("y", self.y[i:i + n], want, i)
            if self.mask is not None:
                _equal("mask", self.mask[i:i + n], _pack(want.float() > 0), i)


A_COUTS = [64, 128, 256, 512, 1024, 2048]
A_CINS = [64, 192, 256, 1088, 4096]
A_SMALL_M = [1, 31, 127, 128, 129, 255, 257]
# (shortcut BN, stats_given): every combination with a shortcut, and none / given without one
MODES = [(False, 0), (False, STATS_GIVEN), (True, 0), (True, STATS_GIVEN), (True, SC_STATS_GIVEN),
         (True, STATS_GIVEN | SC_STATS_GIVEN)]


def _apply_cases():
    out = []
    for a, M in enumerate(A_SMALL_M):
        for b, Cout in enumerate(A_COUTS):
            out.append((A_CINS[(a + b) % len(A_CINS)], Cout, M) + MODES[(a + 2 * b) % len(MODES)])
    out += [(65536, 64, 257) + MODES[2], (65536, 2048, 1000) + MODES[1],   # 1024 K chunks per tile
            (192, 512, 50176) + MODES[5], (4096, 256, 12544) + MODES[4]]
    return out


@gpu
@pytest.mark.usefixtures("memory")
@pytest.mark.parametrize("Cin,Cout,M,shortcut,given", _apply_cases())
def test_bn_add_relu_fwd_exact(Cin, Cout, M, shortcut, given):
    """y, the mask bits, the statistics and the running statistics of both BatchNorms exactly the reference's."""
    _Apply(Cin, Cout, M, M * 3 + Cin + Cout + given, shortcut, given).run()


@gpu
@pytest.mark.usefixtures("memory")
@pytest.mark.parametrize("Cin,Cout,M,shortcut,given", [(64, 64, 1000) + MODES[0], (256, 512, 3001) + MODES[3],
                                                       (1088, 2048, 777) + MODES[5]])
def test_bn_add_relu_fwd_without_mask(Cin, Cout, M, shortcut, given):
    """A NULL mask (the key encoder's call): y as with one."""
    _Apply(Cin, Cout, M, M + Cin, shortcut, given, mask=False).run()


def _slices(Cout):
    return Cout // (128 if Cout % 128 == 0 else 64)


def _apply_plan(M, Cout, sms):
    """launch_apply's grid (csrc/conv1x1_sm90.cu): (m_tiles, tiles per CTA, R)."""
    m_tiles = -(-M // 128)
    R = max(1, sms // _slices(Cout))
    ppc = -(-m_tiles // R)
    return m_tiles, ppc, -(-m_tiles // ppc)


def _apply_edge(kind, Cout, sms):
    """M at an edge of the apply plan: fewer tiles than CTAs, a last CTA with a single tile (itself one row), or
    every CTA full with a ragged last tile."""
    R0 = max(1, sms // _slices(Cout))
    if kind == "few":
        return max(1, R0 - 2) * 128 + 77
    if kind == "ragged":
        return 2 * R0 * 128 - 1
    m = R0 + 1
    while True:
        _, ppc, R = _apply_plan(m * 128, Cout, sms)
        if m - (R - 1) * ppc == 1:
            return (m - 1) * 128 + 1
        m += 1


@gpu
@pytest.mark.usefixtures("memory")
@pytest.mark.parametrize("kind", ["few", "single", "ragged"])
@pytest.mark.parametrize("Cout", [64, 256, 2048])
def test_bn_add_relu_fwd_plan_edges(Cout, kind):
    """M at the apply plan's edges for the SM count of this device."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    M = _apply_edge(kind, Cout, sms)
    m_tiles, ppc, R = _apply_plan(M, Cout, sms)
    if kind == "few":
        assert m_tiles < sms // _slices(Cout)
    if kind == "single":
        assert m_tiles - (R - 1) * ppc == 1 and M % 128 == 1
    k = ["few", "single", "ragged"].index(kind) + [64, 256, 2048].index(Cout)
    _Apply(64 * (1 + k % 3), Cout, M, M + Cout, *MODES[k % len(MODES)]).run()


@gpu
@pytest.mark.usefixtures("memory")
def test_bn_add_relu_fwd_past_4gb():
    """Cout = 2048, Cin = 64 at M = 1,048,705: r and y are 4.3 GB each, offsets past 2^32 bytes."""
    _Apply(64, 2048, 1048705, 11, False, STATS_GIVEN).run()


# ---- one workspace, and CUDA graphs

@gpu
@pytest.mark.usefixtures("memory")
def test_one_workspace_in_turn():
    """moco_conv1x1_bn_stats (Cout = 4096, 64 slabs), the dgrad at C = 2048 then 128, and the apply computing its
    statistics (Cout = 64) on one workspace zeroed once: each call matches its own reference, so each kernel re-arms
    the slab counters the next one uses."""
    L = _lib()
    lib = L.load()
    dev = torch.device("cuda:0")
    ws = torch.zeros(max(lib.moco_conv1x1_workspace_bytes(), lib.moco_bn_workspace_bytes()), dtype=torch.uint8,
                     device=dev)
    _Case(256, 4096, 50176, seed=91).run(ws=ws)
    _Dgrad(2048, 64, 50176, seed=92).run(ws)
    _Dgrad(128, 192, 20000, seed=93).run(ws)
    _Apply(64, 64, 50176, 94, False, 0).run(ws)
    _Dgrad(256, 64, 30001, seed=95).run(ws)


@gpu
@pytest.mark.usefixtures("memory")
def test_dgrad_graph_replay():
    """The dgrad + moco_bn_bwd_apply_given pair captured once and replayed on refreshed inputs."""
    case = _Dgrad(512, 320, 20000, seed=81)
    ws = _new_ws(case.x.device)
    case.run(ws)                                     # warm-up: the kernel attributes are set outside the capture
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        case.launch(ws)
    for _ in range(3):
        case.fill()
        graph.replay()
        torch.cuda.synchronize()
        case.check(case.gout, case.dbeta, case.dgamma, case.dx)


@gpu
@pytest.mark.usefixtures("memory")
def test_apply_graph_replay():
    """The forward computing its statistics captured once and replayed on refreshed inputs: num_batches_tracked
    advances once per replay."""
    case = _Apply(192, 256, 20000, 82, True, 0)
    L = _lib()
    lib = L.load()
    ws = torch.zeros(max(lib.moco_conv1x1_workspace_bytes(), lib.moco_bn_workspace_bytes()), dtype=torch.uint8,
                     device=case.x.device)
    case.run(ws)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        case.launch(ws)
    nbt0 = int(case.bn.stats[2])
    for k in range(3):
        case.fill_x()
        before = case.snapshots()
        graph.replay()
        torch.cuda.synchronize()
        case.check(before, 0.1, 1e-5)
        assert int(case.bn.stats[2]) == nbt0 + k + 1
        assert int(case.sc.stats[2]) == nbt0 + k + 1


# ---- the reference helpers, by hand (no GPU)

def test_plans_by_hand():
    """bn_bwd_reduce_plan (unroll 4) and launch_apply's grid on cases computed by hand."""
    assert _plan(802816, 256, 4) == (25088, 384, 66)       # 4 slabs: R <= 66; ceil(25088 / 66) = 381 -> 384
    assert _plan(50176, 2048, 4) == (1568, 196, 8)         # 32 slabs: 8 CTAs of 6272 rows (49 tiles)
    assert _plan(524545, 128, 4) == (16393, 128, 129)      # 2 slabs: ceil(16393 / 132) = 125 -> 128 passes
    assert _plan(1, 128, 4) == (1, 4, 1)
    assert _r_changes(2048, 1100, 4) == [1, 129, 257, 385, 513, 641, 769, 897, 1025]
    assert _planted(300, 2048, 4) == [127, 128, 255, 256, 277, 299]
    assert _apply_plan(1000, 64, 132) == (8, 1, 8)
    assert _apply_plan(802816, 2048, 132) == (6272, 784, 8)
    assert _apply_plan(265 * 128, 256, 132) == (265, 5, 53)
    assert _apply_edge("single", 64, 132) == 16897          # 133 tiles: 66 CTAs of 2, the 67th one tile of one row
    assert _apply_edge("few", 2048, 132) == 6 * 128 + 77   # 7 tiles on 8 CTAs per slice
    assert _apply_edge("single", 2048, 114) == 1025         # 7 CTAs per slice: 9 tiles -> 2 per CTA, 5 CTAs
    assert _apply_plan(1025, 2048, 114) == (9, 2, 5)


def test_fma32_against_fractions():
    """_fma32 equals the exactly rounded fmaf on 10^4 random triples (a quarter of them cancelling) and on float32
    ties pushed off by less than a float64 ulp, where rounding a float64 sum would be wrong."""
    rng = np.random.default_rng(7)
    n = 10000
    a, b, c = ((rng.standard_normal(n) * 2.0 ** rng.integers(-20, 20, n)).astype(np.float32) for _ in range(3))
    c[::4] = -(a[::4] * b[::4])                            # the float32 product: a * b + c is its rounding error
    got = _fma32(torch.from_numpy(a), torch.from_numpy(b), torch.from_numpy(c)).numpy()
    want = np.array([_fmaf(*t) for t in zip(a, b, c)], dtype=np.float32)
    assert np.array_equal(got, want), int((got != want).sum())
    ties, naive_wrong = [], 0
    for i in range(1, 40, 2):
        for k in (1, 3):
            x, y = np.float32(1 + i * 2.0 ** -12), np.float32(1 + k * 2.0 ** -12)   # x y: a float32 tie
            for tiny in (0.0, 2.0 ** -60, -(2.0 ** -60), 2.0 ** -75):
                z = np.float32(tiny)
                ties.append((x, y, z))
                naive_wrong += np.float32(float(x) * float(y) + float(z)) != _fmaf(x, y, z)
    a, b, c = (np.array(v, dtype=np.float32) for v in zip(*ties))
    got = _fma32(torch.from_numpy(a), torch.from_numpy(b), torch.from_numpy(c)).numpy()
    want = np.array([_fmaf(*t) for t in ties], dtype=np.float32)
    assert np.array_equal(got, want)
    assert naive_wrong > 0                                  # the ties do separate the two roundings
    # by hand: (1 + 2^-12)^2 = 1 + 2^-11 + 2^-24, a tie: to even 1 + 2^-11; 2^-60 more rounds it up
    t = np.float32(1 + 2.0 ** -12)
    assert _fma32(*(torch.tensor([v]) for v in (t, t, 0.0))).item() == 1 + 2.0 ** -11
    up = _fma32(*(torch.tensor([v], dtype=torch.float32) for v in (t, t, 2.0 ** -60))).item()
    assert up == 1 + 2.0 ** -11 + 2.0 ** -23


def test_bf16_ties_by_hand():
    """torch's bf16 rounding (the references' only bf16 rounding) is to nearest, ties to even, as _round(q, 8)."""
    v = [257.0, 259.0, 255.0, 256.5, 258.0, 261.0, 4093.0, 4088.0, 4104.0, -257.0, -259.0, 1028.0, 1036.0]
    want = [256.0, 260.0, 255.0, 256.0, 258.0, 260.0, 4096.0, 4096.0, 4096.0, -256.0, -260.0, 1024.0, 1040.0]
    got = torch.tensor(v).bfloat16().float().tolist()
    assert got == want
    assert [float(_round(Fraction(x), 8)) for x in v] == want


def test_bwd_coefs_by_hand():
    """bwd_coefs on values whose products are exact: gamma = 2, invstd = 1/2, sums 8 and 4 over M = 4."""
    cA, cB, cD = _bwd_coefs([2.0], [0.5], [0.5], [8.0], [4.0], 4)[:, 0]
    # k1 = 1, m1 = 2, m2 = 1, cB = -1 * 1 * 0.5, cD = fmaf(0.5, 0.5, -2)
    assert (cA, cB, cD) == (np.float32(1.0), np.float32(-0.5), np.float32(-1.75))
    # the fmaf keeps the product's low bits: (1 + 2^-12)^2 - 1 = 2^-11 + 2^-24, not fl32(fl32(a b) - 1) = 2^-11
    t = float(np.float32(1 + 2.0 ** -12))
    assert _fmaf(t, t, -1.0) == np.float32(2.0 ** -11 + 2.0 ** -24)
