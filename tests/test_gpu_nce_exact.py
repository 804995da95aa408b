"""The replicated InfoNCE head (moco_nce_fwd / moco_nce_step / moco_nce_bwd_dense) on exact-arithmetic inputs.

Every q, k and queue row below has 16 nonzero entries of +-1/4 (4 of +-1/2 when C < 16): it is exactly unit-norm and
bf16-representable, and every dot product is a multiple of 1/16 with |dot| <= 1, which fp32 gets exactly in any
summation order (wgmma's included).  So

* the dense logits have one right answer, fp32(fp32(dot) * fp32(inv_T)), and are compared bit for bit;
* lse / loss / prob are compared with a float64 reference at a tolerance that the test itself shows to be smaller
  than the effect of removing or duplicating any one of the planted queue rows (copies of a query, dot = 1) that sit
  at both ends of the queue, on both sides of tile boundaries (BN = 128 and 64) and inside the ragged last tile;
* dq is checked element by element against the bound the header's contract gives (P rounded to bf16 once, fp32
  accumulation), computed in float64 from the reference's softmax.  In the "tagged" variant every entry is
  nonnegative and k = 0, so dq is the queue term inv_T/N sum_j p_ij m_j alone, without cancellation: the bound is
  then a per-coordinate relative check of a few tenths of a percent, and a planted row lost from any slice, tile or
  chunk moves some coordinate by far more.

Each case also asserts, with torch.profiler, which kernels ran, and that _lib.launches counts the same number."""
import collections
import ctypes
import math
import re

import numpy as np
import pytest
import torch

from oracle import moco_oracle as O
from tests import helpers

pytestmark = pytest.mark.gpu

U24 = 2.0 ** -24                  # fp32 unit roundoff
BF16_P = 2.0 ** -8                # relative error of rounding P to bf16 once


def _lib():
    from moco_b200 import _lib
    return _lib


def _sms():
    n = ctypes.c_int()
    assert _lib().load().moco_device_info(ctypes.byref(n), None, None) == 0
    return n.value


# ---------------------------------------------------------------------------------------------------------------
# exact operands
# ---------------------------------------------------------------------------------------------------------------
def _nnz(C):
    return (16, 0.25) if C >= 16 else (4, 0.5)


def exact_rows(rng, n, C, signed=True):
    """n rows with exactly nnz entries of +-val at seeded random positions (all +val when not signed)."""
    nnz, val = _nnz(C)
    out = np.zeros((n, C), np.float32)
    pos = np.argpartition(rng.random((n, C), dtype=np.float32), nnz, axis=1)[:, :nnz]
    v = (rng.integers(0, 2, size=(n, nnz)) * 2 - 1).astype(np.float32) * val if signed else np.full((n, nnz), val, np.float32)
    np.put_along_axis(out, pos, v, axis=1)
    return out


def tagged_rows(seed, n, C):
    """Nonnegative rows whose support is a seeded function of row // 64."""
    nnz, val = _nnz(C)
    out = np.zeros((n, C), np.float32)
    for b in range((n + 63) // 64):
        out[b * 64:(b + 1) * 64, np.random.default_rng([seed, b]).choice(C, nnz, replace=False)] = val
    return out


def plant_positions(K, N):
    """Queue rows that get a copy of a query: both ends, both sides of every 64-row (hence 128-row) tile boundary
    (thinned evenly to at most 4 per query), and inside the ragged last tile of either tile size."""
    bounds = np.arange(64, K, 64)
    if len(bounds) > 4 * N:
        bounds = np.unique(bounds[np.linspace(0, len(bounds) - 1, 4 * N).astype(int)])
    pos = {0, K - 1}
    for b in bounds:
        pos.update((int(b) - 1, int(b)))
    for bn in (64, 128):
        r = K % bn
        if r > 2:
            pos.add(K - 1 - r // 2)
    return sorted(p for p in pos if 0 <= p < K)


def make_case(N, C, K, variant, seed):
    """(q, k, queue, plants): plants = [(query i, queue row j)] with queue[j] == q[i]."""
    rng = np.random.default_rng(seed)
    if variant == "tagged":
        q = exact_rows(rng, N, C, signed=False)
        k = np.zeros((N, C), np.float32)
        queue = tagged_rows(seed, K, C)
    else:
        q, k, queue = exact_rows(rng, N, C), exact_rows(rng, N, C), exact_rows(rng, K, C)
    plants = [(t % N, j) for t, j in enumerate(plant_positions(K, N))]
    for i, j in plants:
        queue[j] = q[i]
    return q, k, queue, plants


# ---------------------------------------------------------------------------------------------------------------
# float64 reference
# ---------------------------------------------------------------------------------------------------------------
def reference(q, k, queue, inv_T, chunk=8192):
    """lse, loss_rows, prob_rows, S = sum_j p_ij m_j and A = sum_j p_ij |m_j| in float64, with the logits scaled by
    the fp32 inv_T the kernels receive."""
    q64, k64 = q.astype(np.float64), k.astype(np.float64)
    K = queue.shape[0]
    x0 = (q64 * k64).sum(1) * inv_T
    lse = x0.copy()
    for j0 in range(0, K, chunk):
        x = q64 @ queue[j0:j0 + chunk].astype(np.float64).T * inv_T
        lse = np.logaddexp(lse, O.logsumexp_rows(x))
    S = np.zeros_like(q64)
    A = np.zeros_like(q64)
    for j0 in range(0, K, chunk):
        m = queue[j0:j0 + chunk].astype(np.float64)
        p = np.exp(q64 @ m.T * inv_T - lse[:, None])
        S += p @ m
        A += p @ np.abs(m)
    return lse, lse - x0, np.exp(x0 - lse), S, A


def lse_tol(lse):
    return 3e-5 + 3e-6 * np.abs(lse)


def gamma(n):
    return n * U24 / (1 - n * U24)


def dq_expected_and_bound(k, inv_T, N, K, prob, tol, S, A):
    """dq = inv_T/N ((p0 - 1) k + S) and its per-element bound: P rounded to bf16 once (2^-8), fp32 accumulation
    over K rows (gamma_K), p itself off by the lse error (tol), the final fp32 roundings, and fp32's range: terms
    below 2^-126 flush to zero (queue entries are at most 1 here)."""
    k64 = np.abs(k.astype(np.float64))
    g = inv_T / N
    eps = (2 * tol + 1e-5)[:, None]
    exp = g * ((prob - 1.0)[:, None] * k.astype(np.float64) + S)
    bound = g * ((BF16_P + gamma(K + 8) + eps) * A + (eps * prob[:, None] + 4 * U24) * k64 + (K + 2) * 2.0 ** -126) + \
        4 * U24 * np.abs(exp)
    return exp, bound


def assert_planted_rows_matter(lse, inv_T, plants, tol):
    """Removing (or duplicating) any planted row moves its query's lse by more than the tolerance."""
    for i, _ in plants:
        dup = math.log1p(math.exp(inv_T - lse[i]))           # the planted logit is 1 * inv_T
        assert dup > tol[i], (i, dup, tol[i])


# ---------------------------------------------------------------------------------------------------------------
# calling the head and watching which kernels ran
# ---------------------------------------------------------------------------------------------------------------
_KERNELS = ("prep_kernel", "combine_kernel", "dq_reduce_kernel", "nce_tail_kernel", "simt_rows_kernel",
            "enqueue_kernel", "enqueue_scalar_kernel", "bwd_dense_kernel", "f32_to_bf16_kernel")
_MODES = {"0": "fused", "1": "normed", "2": "stats"}


def _kernel_label(name):
    m = re.search(r"nce_sweep_kernel<(\d+), *(\d+), *(\d+)>", name) or \
        re.search(r"nce_sweep_kernelILi(\d+)ELi(\d+)ELi(\d+)E", name)
    if m:
        return f"sweep_{_MODES[m.group(2)]}_cl{m.group(3)}"
    for kname in _KERNELS:
        if re.search(rf"\b{kname}\b", name) or f"{len(kname)}{kname}" in name:
            return kname
    return None


def profiled(fn, reset=None):
    """(result of fn(), Counter of this library's kernels that ran, _lib.launches delta): tests.helpers.profiled."""
    out, kernels, counted = helpers.profiled([fn], reset)[0]
    return out, collections.Counter(l for l in map(_kernel_label, kernels) if l is not None), counted


def expected_kernels(N, C, inv_T, flags, want_dq, want_logits, f32):
    lib = _lib()
    tc = not (flags & lib.NCE_FORCE_SIMT) and C % 64 == 0 and C <= 256 and (N + 127) // 128 <= _sms()
    if not tc:
        return collections.Counter({"prep_kernel": 1, "simt_rows_kernel": 1})
    one = want_dq and not want_logits and not (flags & lib.NCE_TWO_PASS) and \
        ((flags & lib.NCE_ONE_PASS) or inv_T <= lib.ONE_PASS_MAX_INV_T)
    if one:
        c = collections.Counter({"sweep_fused_cl1": 1, "nce_tail_kernel": 1})
        if C > 128 and f32:
            c["prep_kernel"] = 1
        return c
    cl = 2 if flags & lib.NCE_CTA_PAIR else 1
    c = collections.Counter({"prep_kernel": 1, f"sweep_stats_cl{cl}": 1, "combine_kernel": 1})
    if want_dq:
        c.update({"sweep_normed_cl1": 1, "dq_reduce_kernel": 1})
    return c


class Head:
    """Device buffers for one moco_nce_fwd call on numpy operands."""

    def __init__(self, q, k, queue, dtype):
        self.N, self.C = q.shape
        self.K = queue.shape[0]
        self.q = torch.from_numpy(q).cuda().to(dtype)
        self.k = torch.from_numpy(k).cuda().to(dtype)
        self.queue = torch.from_numpy(queue).cuda().bfloat16()
        lib = _lib().load()
        self.ws_bytes = int(lib.moco_nce_workspace_bytes(self.N, self.C, self.K))
        self.ws = torch.empty(self.ws_bytes + 256, dtype=torch.uint8, device="cuda")
        self.ws_ptr = self.ws.data_ptr() + (-self.ws.data_ptr()) % 256

    def fwd(self, inv_T, flags, want_logits, want_dq):
        L = _lib()
        lib = L.load()
        f = dict(dtype=torch.float32, device="cuda")
        out = {"lse": torch.empty(self.N, **f), "loss_rows": torch.empty(self.N, **f),
               "prob_rows": torch.empty(self.N, **f), "loss_prob": torch.empty(2, **f),
               "logits": torch.empty(self.N, self.K + 1, **f) if want_logits else None,
               "dq": torch.empty(self.N, self.C, **f) if want_dq else None}
        ptr = lambda t: t.data_ptr() if t is not None else None
        rc = lib.moco_nce_fwd(self.q.data_ptr(), self.k.data_ptr(), L.dtype_code(self.q), self.queue.data_ptr(),
                              self.N, self.C, self.K, inv_T, ptr(out["logits"]), ptr(out["lse"]),
                              ptr(out["loss_rows"]), ptr(out["prob_rows"]), ptr(out["loss_prob"]), ptr(out["dq"]),
                              self.ws_ptr, self.ws_bytes, flags, L.cur_stream())
        L.check(rc, "moco_nce_fwd")
        return out


def _flag(name):
    L = _lib()
    return {"auto": L.NCE_AUTO, "onepass": L.NCE_ONE_PASS, "twopass": L.NCE_TWO_PASS,
            "tc1": L.NCE_SINGLE_CTA | L.NCE_TWO_PASS, "tc2": L.NCE_CTA_PAIR | L.NCE_TWO_PASS,
            "simt": L.NCE_FORCE_SIMT}[name]


def _fp32_inv_T(T):
    return float(np.float32(1.0 / T))


def check_stats(out, lse, loss_rows, prob_rows, tol):
    lse_g = out["lse"].cpu().numpy().astype(np.float64)
    assert np.isfinite(lse_g).all()
    err = np.abs(lse_g - lse)
    assert (err <= tol).all(), (err.max(), int(err.argmax()))
    assert (np.abs(out["loss_rows"].cpu().numpy() - loss_rows) <= tol + 4e-6 * np.abs(loss_rows)).all()
    prob_g = out["prob_rows"].cpu().numpy().astype(np.float64)
    assert (np.abs(prob_g - prob_rows) <= prob_rows * (tol + 1e-6) + 1e-12).all()
    lp = out["loss_prob"].cpu().numpy().astype(np.float64)
    assert abs(lp[0] - loss_rows.mean()) <= tol.mean() + 4e-6 * abs(loss_rows.mean()) + 1e-6
    assert abs(lp[1] - prob_rows.mean()) <= (prob_rows * (tol + 1e-6)).mean() + 1e-6 * prob_rows.mean() + 1e-9


# ---------------------------------------------------------------------------------------------------------------
# dense logits, bit for bit
# ---------------------------------------------------------------------------------------------------------------
DENSE = [  # (N, C, K, flag)
    (1, 64, 1, "tc1"), (1, 64, 1, "simt"), (63, 128, 127, "tc1"), (65, 192, 129, "tc1"), (130, 256, 65, "tc2"),
    (128, 128, 126689, "tc1"), (127, 256, 126689, "tc2"),                 # ragged K, CTA pair with ragged N
    (129, 128, 131 * 128 - 5, "tc1"), (64, 256, 133 * 64 + 3, "tc1"),     # num_tiles just under / over #SM
    (128, 192, 16384, "tc2"), (2048, 64, 16384, "auto"),
    (63, 8, 1000, "auto"), (65, 96, 129, "auto"), (130, 100, 4097, "auto"), (13, 1000, 300, "auto"),
    (64, 128, 1000, "simt"), (16897, 128, 64, "auto"),                    # N > 128 * #SM: the CUDA-core kernel
]


@pytest.mark.parametrize("N,C,K,flag", DENSE)
def test_dense_logits_are_exact(N, C, K, flag):
    T = 0.07
    inv_T = _fp32_inv_T(T)
    q, k, queue, plants = make_case(N, C, K, "signed", seed=N * 7 + C + K)
    h = Head(q, k, queue, torch.float32)
    flags = _flag(flag)
    out, ran, counted = profiled(lambda: h.fwd(inv_T, flags, True, False))
    assert ran == expected_kernels(N, C, inv_T, flags, False, True, True), ran
    assert counted == sum(ran.values())
    got = out["logits"]
    # expected, in fp32 from the exact float64 dot: column 0 = <q, k> * inv_T, columns 1.. = <q, queue_j> * inv_T
    inv32 = np.float32(inv_T)
    exp0 = ((q.astype(np.float64) * k.astype(np.float64)).sum(1)).astype(np.float32) * inv32
    np.testing.assert_array_equal(got[:, 0].cpu().numpy(), exp0)
    q64 = q.astype(np.float64)
    for j0 in range(0, K, 16384):
        dots = (q64 @ queue[j0:j0 + 16384].astype(np.float64).T).astype(np.float32)
        np.testing.assert_array_equal(got[:, 1 + j0:1 + j0 + 16384].cpu().numpy(), dots * inv32)
    lse, loss_rows, prob_rows, _, _ = reference(q, k, queue, inv_T)
    tol = lse_tol(lse)
    assert_planted_rows_matter(lse, inv_T, plants, tol)
    check_stats(out, lse, loss_rows, prob_rows, tol)


# ---------------------------------------------------------------------------------------------------------------
# lse / loss / prob and the queue term of dq
# ---------------------------------------------------------------------------------------------------------------
GRAD = [  # (N, C, K, dtype, flag, T, variant)
    (64, 128, 16384, "bf16", "onepass", 0.07, "tagged"),
    (64, 256, 16384, "f32", "onepass", 0.07, "tagged"),                  # + the bf16 copy of q
    (128, 192, 16384, "bf16", "onepass", 0.07, "signed"),
    (129, 64, 127, "bf16", "onepass", 0.03, "tagged"),
    (256, 64, 262144, "bf16", "onepass", 0.07, "tagged"),
    (128, 128, 262144, "f32", "auto", 0.07, "signed"),
    (2048, 128, 16384, "f32", "twopass", 0.03, "tagged"),
    (130, 192, 126689, "f32", "twopass", 0.07, "signed"),
    (65, 256, 133 * 64 + 3, "bf16", "tc2", 0.03, "tagged"),              # CTA-pair statistics, then the dq pass
    (127, 128, 131 * 128 - 5, "f32", "auto", 0.03, "signed"),            # T = 0.03: AUTO takes two passes
    (1, 64, 1, "f32", "auto", 0.07, "signed"),
    (63, 64, 65, "bf16", "twopass", 0.07, "tagged"),
    (16896, 64, 128, "bf16", "onepass", 0.07, "signed"),                 # the largest N of the one sweep
    (16897, 128, 65, "f32", "auto", 0.07, "tagged"),                     # beyond it: prep + CUDA-core rows
    (16897, 256, 129, "f32", "twopass", 0.03, "signed"),
    (63, 8, 1000, "f32", "auto", 0.07, "tagged"),                        # C % 64 != 0: CUDA-core rows
    (64, 100, 4097, "f32", "auto", 0.07, "tagged"),
    (127, 1000, 300, "bf16", "auto", 0.03, "signed"),
    (65, 96, 129, "bf16", "simt", 0.03, "tagged"),
    (130, 128, 1000, "f32", "simt", 0.07, "tagged"),
]


@pytest.mark.parametrize("N,C,K,dtype,flag,T,variant", GRAD)
def test_loss_and_queue_term_of_dq(N, C, K, dtype, flag, T, variant):
    inv_T = _fp32_inv_T(T)
    q, k, queue, plants = make_case(N, C, K, variant, seed=N * 3 + C * 5 + K)
    h = Head(q, k, queue, torch.float32 if dtype == "f32" else torch.bfloat16)
    flags = _flag(flag)
    out, ran, counted = profiled(lambda: h.fwd(inv_T, flags, False, True))
    assert ran == expected_kernels(N, C, inv_T, flags, True, False, dtype == "f32"), ran
    assert counted == sum(ran.values())
    lse, loss_rows, prob_rows, S, A = reference(q, k, queue, inv_T)
    tol = lse_tol(lse)
    assert_planted_rows_matter(lse, inv_T, plants, tol)
    check_stats(out, lse, loss_rows, prob_rows, tol)
    exp, bound = dq_expected_and_bound(k, inv_T, N, K, prob_rows, tol, S, A)
    dq = out["dq"].cpu().numpy().astype(np.float64)
    err = np.abs(dq - exp)
    bad = err > bound
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:5].tolist(), float((err / np.maximum(bound, 1e-30)).max()))
    if variant == "tagged":
        # no cancellation: the bound is a per-coordinate relative check at 2^-8 + gamma_K + the lse tolerance
        nz = exp > 0
        assert (bound[nz] / exp[nz]).max() < BF16_P + gamma(K + 8) + 2 * tol.max() + 1e-4
        # and a planted row is more than twice the bound at some coordinate: losing it could not pass
        for i, j in plants[:64]:
            share = np.exp(inv_T - lse[i]) * queue[j].astype(np.float64) * inv_T / N
            c = int(np.argmax(share))
            assert share[c] > 2 * bound[i, c], (i, j, share[c] / bound[i, c])


def test_tensor_core_flags_beyond_the_envelope_are_an_error():
    """SINGLE_CTA / CTA_PAIR demand the tensor-core kernels: with more 128-row (CTA pair: 256-row) blocks of q than
    SMs they fail loudly instead of falling back to the CUDA-core kernel."""
    N = 128 * _sms() + 1
    q, k, queue, _ = make_case(N, 64, 64, "signed", seed=N)
    h = Head(q, k, queue, torch.bfloat16)
    for flag in ("tc1", "tc2"):
        with pytest.raises(RuntimeError, match="statistics kernel"):
            h.fwd(_fp32_inv_T(0.07), _flag(flag), False, True)


def test_grad_matrix_covers_every_flag_dtype_and_temperature():
    """The matrix above runs every flag of the header at least once, fp32 and bf16, both temperatures."""
    assert {g[4] for g in GRAD} >= {"auto", "onepass", "twopass", "tc2", "simt"}
    assert {g[3] for g in GRAD} == {"f32", "bf16"} and {g[5] for g in GRAD} == {0.07, 0.03}


# ---------------------------------------------------------------------------------------------------------------
# in-kernel normalisation with norms from 2^-10 to 2^10 (exact: the norms are powers of two)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,dtype", [(64, "f32"), (128, "bf16"), (128, "f32")])
def test_normalize_is_exact_for_any_input_norm(C, dtype):
    L = _lib()
    lib = L.load()
    N, K, T = 96, 4160, 0.07
    inv_T = _fp32_inv_T(T)
    rng = np.random.default_rng(C)
    q, k, queue, plants = make_case(N, C, K, "signed", seed=C + 1)
    kall = exact_rows(rng, N, C)
    sq = 2.0 ** rng.integers(-10, 11, size=N)
    sk = 2.0 ** rng.integers(-10, 11, size=N)
    sa = 2.0 ** rng.integers(-10, 11, size=N)
    tdt = torch.float32 if dtype == "f32" else torch.bfloat16
    xq = torch.from_numpy((q * sq[:, None]).astype(np.float32)).cuda().to(tdt)
    xk = torch.from_numpy((k * sk[:, None]).astype(np.float32)).cuda().to(tdt)
    xa = torch.from_numpy((kall * sa[:, None]).astype(np.float32)).cuda().to(tdt)
    qb = torch.from_numpy(queue).cuda().bfloat16()
    qf = torch.from_numpy(queue).cuda()
    f = dict(dtype=torch.float32, device="cuda")
    lse_t, lr, pr, lp, dq = (torch.empty(N, **f), torch.empty(N, **f), torch.empty(N, **f), torch.empty(2, **f),
                             torch.empty(N, C, **f))
    ws_bytes = int(lib.moco_nce_workspace_bytes(N, C, K))
    ws = torch.empty(ws_bytes + 256, dtype=torch.uint8, device="cuda")
    index = K - 40                                       # the enqueue wraps past K - 1
    call = lambda: L.check(lib.moco_nce_step(
        xq.data_ptr(), xk.data_ptr(), L.dtype_code(xq), 1, qb.data_ptr(), qf.data_ptr(), N, C, K, inv_T,
        xa.data_ptr(), L.dtype_code(xa), N, index, None, lse_t.data_ptr(), lr.data_ptr(), pr.data_ptr(), lp.data_ptr(),
        dq.data_ptr(), ws.data_ptr() + (-ws.data_ptr()) % 256, ws_bytes, L.NCE_ONE_PASS, L.cur_stream()), "moco_nce_step")
    _, ran, counted = profiled(call, reset=lambda: (qb.copy_(torch.from_numpy(queue).cuda().bfloat16()),
                                                    qf.copy_(torch.from_numpy(queue).cuda())))
    assert ran == collections.Counter({"sweep_fused_cl1": 1, "nce_tail_kernel": 1}) and counted == 2, ran
    lse, loss_rows, prob_rows, S, A = reference(q, k, queue, inv_T)
    tol = lse_tol(lse)
    assert_planted_rows_matter(lse, inv_T, plants, tol)
    check_stats({"lse": lse_t, "loss_rows": lr, "prob_rows": pr, "loss_prob": lp}, lse, loss_rows, prob_rows, tol)
    g, B = dq_expected_and_bound(k, inv_T, N, K, prob_rows, tol, S, A)        # gradient w.r.t. the unit q
    qh = q.astype(np.float64)
    proj = (qh * g).sum(1, keepdims=True)
    exp = (g - qh * proj) / sq[:, None]
    bound = (B + np.abs(qh) * (np.abs(qh) * B).sum(1, keepdims=True) +
             4 * U24 * (np.abs(g) + np.abs(qh * proj))) / sq[:, None] + 4 * U24 * np.abs(exp)
    err = np.abs(dq.cpu().numpy().astype(np.float64) - exp)
    assert (err <= bound).all(), float((err / bound).max())
    # the enqueued rows are the normalised keys, exactly
    ids = (np.arange(N) + index) % K
    want = queue.copy()
    want[ids] = kall
    np.testing.assert_array_equal(qf.cpu().numpy(), want)
    np.testing.assert_array_equal(qb.float().cpu().numpy(), want)


# ---------------------------------------------------------------------------------------------------------------
# the exact CUDA-core fallback reads the queue BEFORE the fused enqueue overwrites it
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("device_index", [False, True])
def test_exact_fallback_reads_the_slots_the_fused_enqueue_overwrites(device_index):
    """q has norm 12, so its logits against its own direction (12 / T) overflow the one-sweep kernel's partial sums
    and every row is recomputed exactly on CUDA cores by the tail kernel, which also enqueues.  Each query's direction
    is ONLY in the ring slots this step's enqueue overwrites ([index, index + n_all), wrapping past K - 1): if an
    enqueue block wrote before the row blocks had finished reading, those rows would see the new keys instead."""
    from moco_b200.NCE import MemoryMoCo
    L = _lib()
    N, C, K, T = 64, 128, 4096, 0.07
    rng = np.random.default_rng(31)
    u = exact_rows(rng, N, C)
    q = u * 12.0                                        # 16 entries of +-3: bf16-representable, norm exactly 12
    k = exact_rows(rng, N, C)
    k_all = exact_rows(rng, N, C)
    queue = exact_rows(rng, K, C)
    index = K - 24
    ids = (np.arange(N) + index) % K
    queue[ids] = u                                      # query i's direction sits in the slot key i will take
    inv_T = _fp32_inv_T(T)
    lse, loss_rows, prob_rows, S, A = reference(q, k, queue, inv_T)
    mod = MemoryMoCo(C, K, T, device_index=device_index)
    mod.memory.copy_(torch.from_numpy(queue))
    mod = mod.cuda()
    mod.kernel_flags = L.NCE_ONE_PASS
    mod.index = index
    mod._queue_bf16()
    qt = torch.from_numpy(q).cuda().requires_grad_(True)

    def step():
        l, p = mod.forward_loss(qt, torch.from_numpy(k).cuda(), torch.from_numpy(k_all).cuda())
        l.backward()
        return l, p

    def reset():
        mod.memory.copy_(torch.from_numpy(queue).cuda())
        mod._queue_bf16()
        mod.index = index
        qt.grad = None
    (l, p), ran, counted = profiled(step, reset)
    assert ran == collections.Counter({"sweep_fused_cl1": 1, "nce_tail_kernel": 1}) and counted == 2, ran
    tol = lse_tol(lse)
    assert abs(float(l) - loss_rows.mean()) <= tol.mean() + 4e-6 * abs(loss_rows.mean())
    assert abs(float(p) - prob_rows.mean()) <= (prob_rows * (tol + 1e-6)).mean() + 1e-12
    lse_g = mod._scratch[(N, C, K, qt.device)].lse.cpu().numpy()
    assert (np.abs(lse_g - lse) <= tol).all()
    # a single planted direction already moves lse far beyond the tolerance
    assert (np.log1p(np.exp(12 * inv_T - lse)) > tol).all()
    exp, bound = dq_expected_and_bound(k, inv_T, N, K, prob_rows, tol, S, A)
    assert (np.abs(qt.grad.cpu().numpy() - exp) <= bound).all()
    want = queue.copy()
    want[ids] = k_all
    np.testing.assert_array_equal(mod.memory.cpu().numpy(), want)
    np.testing.assert_array_equal(mod.memory_bf16.float().cpu().numpy(), want)
    assert mod.index == (index + N) % K
    if device_index:
        assert mod.sync_index() == (index + N) % K


# ---------------------------------------------------------------------------------------------------------------
# device-side ring index on every path
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,T,grad", [(128, 0.03, True), (96, 0.07, True), (192, 0.07, True), (128, 0.07, False)],
                         ids=["two-pass", "cuda-core", "c192-one-sweep", "no-grad"])
def test_device_index_equals_host_index_on_every_path(C, T, grad):
    """MemoryMoCo(device_index=True) outside the one-sweep path with the fused enqueue: T = 0.03 (two passes), C = 96
    (CUDA-core rows), C = 192 (one sweep, separate enqueue kernel) and no gradient (statistics pass only).  Same loss,
    prob, dq and queue as device_index=False, step after step across the ring's end, and sync_index() returns the
    host's position."""
    from moco_b200.NCE import MemoryMoCo
    N, K, steps = 64, 200, 5
    rng = np.random.default_rng(C + int(grad))
    queue = exact_rows(rng, K, C)
    mods = []
    for dev in (False, True):
        m = MemoryMoCo(C, K, T, device_index=dev)
        m.memory.copy_(torch.from_numpy(queue))
        mods.append(m.cuda())
    orc = O.MemoryMoCoOracle(queue, T)
    for s in range(steps):
        q, k = exact_rows(rng, N, C), exact_rows(rng, N, C)
        res = []
        for m in mods:
            qt = torch.from_numpy(q).cuda().requires_grad_(grad)
            kt = torch.from_numpy(k).cuda()
            if grad:
                l, p = m.forward_loss(qt, kt, kt)
                l.backward()
                res.append((float(l), float(p), qt.grad.cpu().numpy()))
            else:
                with torch.no_grad():
                    l, p = m.forward_loss(qt, kt, kt)
                res.append((float(l), float(p), None))
        assert res[0][:2] == res[1][:2], s
        if grad:
            np.testing.assert_array_equal(res[0][2], res[1][2])
        orc.enqueue(k)
        assert torch.equal(mods[0].memory, mods[1].memory), s
        np.testing.assert_array_equal(mods[1].memory.cpu().numpy(), orc.memory)
        assert mods[1].sync_index() == mods[0].index == orc.index, s
    assert (steps * N) > K                              # the ring wrapped


def test_device_index_persists_the_device_position():
    """persist_index + device_index at C = 192: state_dict() syncs the index from the device copy."""
    from moco_b200.NCE import MemoryMoCo
    N, C, K, T = 64, 192, 150, 0.07
    rng = np.random.default_rng(5)
    m = MemoryMoCo(C, K, T, persist_index=True, device_index=True).cuda()
    for _ in range(3):
        q = torch.from_numpy(exact_rows(rng, N, C)).cuda().requires_grad_(True)
        l, _ = m.forward_loss(q, q.detach(), q.detach())
        l.backward()
    assert int(m.state_dict()["params"]) == (3 * N) % K == m.index


# ---------------------------------------------------------------------------------------------------------------
# moco_nce_bwd_dense called directly
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k_dtype", ["f32", "bf16"])
@pytest.mark.parametrize("N,C,K", [(13, 100, 1000), (9, 512, 300), (8, 1024, 129)])
def test_bwd_dense_within_its_accumulation_bound(N, C, K, k_dtype):
    """dq_i = inv_T (g_i0 k_i + sum_j g_ij queue_j) for an arbitrary fp32 g: grid.y > 1 (C > 256), C not a multiple
    of 32, N not a multiple of 8.  Each element within gamma_K sum_j |g_ij| |m_jc| plus the k term's roundings."""
    L = _lib()
    lib = L.load()
    T = 0.07
    inv_T = _fp32_inv_T(T)
    rng = np.random.default_rng(N * C + K)
    g = rng.standard_normal((N, K + 1)).astype(np.float32)
    k = O.bf16_round(rng.standard_normal((N, C)).astype(np.float32))
    queue = O.bf16_round(rng.standard_normal((K, C)).astype(np.float32))
    gt = torch.from_numpy(g).cuda()
    kt = torch.from_numpy(k).cuda().to(torch.float32 if k_dtype == "f32" else torch.bfloat16)
    qb = torch.from_numpy(queue).cuda().bfloat16()
    dq = torch.empty(N, C, dtype=torch.float32, device="cuda")
    call = lambda: L.check(lib.moco_nce_bwd_dense(gt.data_ptr(), kt.data_ptr(), L.dtype_code(kt), qb.data_ptr(), N, C,
                                                  K, inv_T, dq.data_ptr(), L.cur_stream()), "moco_nce_bwd_dense")
    _, ran, counted = profiled(call)
    assert ran == collections.Counter({"bwd_dense_kernel": 1}) and counted == 1, ran
    g64, k64, m64 = g.astype(np.float64), k.astype(np.float64), queue.astype(np.float64)
    exp = inv_T * (g64[:, :1] * k64 + g64[:, 1:] @ m64)
    bound = inv_T * gamma(K + 4) * (np.abs(g64[:, 1:]) @ np.abs(m64) + np.abs(g64[:, :1] * k64)) + 2 * U24 * np.abs(exp)
    err = np.abs(dq.cpu().numpy().astype(np.float64) - exp)
    assert (err <= bound).all(), float((err / bound).max())
    # the bound is tight enough that a dropped queue row (first, chunk end, last) could not hide in it
    for j in sorted({0, min(127, K - 1), K - 1}):
        assert (inv_T * np.abs(g64[:, 1 + j, None] * m64[j][None]) > 2 * bound).mean() > 0.5, j
