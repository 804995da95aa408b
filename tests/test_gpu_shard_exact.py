"""The sharded-queue head (moco_nce_shard_stats / _merge / _dq / _dq_finish / _dq_finish_peers) on exact-arithmetic
inputs, one shard's partials at a time.

q, k and the queue are the exact rows of test_gpu_nce_exact (16 nonzero entries of +-1/4): every dot product is a
multiple of 1/16 and exact in any summation order.  The queue is split into W shards of Ks rows, and every shard gets
copies of queries (dot = 1) at rows 0 and Ks - 1, on both sides of its 64- and 128-row tile boundaries and inside its
ragged last tile; every rank's queries are planted, and for W >= 2 some sit in another rank's shard.  Each link of
the chain is then checked against float64 on its own:

1. rank r's (max, sum) pair: ms.x + log2(ms.y) against the float64 log2 of sum_{j in shard r} 2^(x_ij log2e).  This
   form holds for the two-pass pair, the one-sweep pair (constant stabiliser, sum) and the exact-row pair (lse2, 1).
   The tolerance is lse_tol in the log2 domain, and the test shows it to be smaller than the effect of removing or
   duplicating any one planted row of that shard;
2. the merge: lse, loss_rows and prob_rows within lse_tol, loss_prob as the means over all Nq rows, every rank's merge
   bit-identical, and the planted rows shown to matter;
3. rank r's o_partial against sum_{j in shard r} exp(x_ij - lse_i) shard_j with the bound of dq_expected_and_bound
   (P rounded to bf16 once, fp32 accumulation over Ks rows, the lse error).  In the "tagged" variant (entries >= 0,
   k = 0) that bound is a per-coordinate relative check, and a planted row's share exceeds twice it;
4. the finish: moco_nce_shard_dq_finish on the rank-order sum of the o_partial blocks and
   moco_nce_shard_dq_finish_peers on the peer table agree bit for bit, and both equal the fp32 restatement below;
   dq is then within dq_expected_and_bound of the float64 gradient.

The restatement follows the SASS of both finish kernels (cuobjdump -sass, nvcc 12.9, -O3, sm_90a, no fast-math):
dq_reduce_kernel (finish mode) and dq_finish_peers_kernel both compute
    gscale = inv_T / (float)N                      IEEE division (FCHK + MUFU.RCP refinement with the slow path)
    acc    = ((0 + o_0) + o_1) + ... + o_{W-1}     FADD in rank order (dq_reduce_kernel: the summed o plus zeros)
    dq     = FMUL(FFMA(FADD(prob, -1), k, acc), gscale)
so pm1 * k + acc is one fused multiply-add and the product with gscale is a separate rounding.

A second test moves a few q rows to power-of-two norms and plants a partner row in one shard only, so that in
one-sweep mode those rows leave the kernel's safe range on that shard and stay inside it on the others: the merge
then combines exact (lse2, 1) pairs with ordinary pairs for the same row, and every check above still holds.  The
envelope test runs the largest Nq = W * N the statistics kernels accept (derived from the launchers' rule
mblks * G <= #SM) exactly, and one row more must be refused with MOCO_ERR_UNSUPPORTED.  Every case stays under 10 GB
of device memory (asserted)."""
import gc
import math
import sys

import numpy as np
import pytest
import torch

from tests.test_gpu_nce_exact import (BF16_P, _fp32_inv_T, _sms, assert_planted_rows_matter, check_stats,
                                      dq_expected_and_bound, exact_rows, gamma, lse_tol, plant_positions, reference,
                                      tagged_rows)
from tests.test_gpu_shard_sim import _workspace, simulate

pytestmark = pytest.mark.gpu

MEM_LIMIT = 10 * 2 ** 30
LN2 = math.log(2.0)
MOCO_ERR_UNSUPPORTED = -2
FLAGS = {"one_pass": 1024, "two_pass": 0, "cta_pair": 2}      # MOCO_NCE_ONE_PASS, the default two passes, CTA_PAIR


def _lib():
    from moco_b200 import _lib
    return _lib


@pytest.fixture(autouse=True)
def memory():
    """Each case under MEM_LIMIT bytes of device memory; its tensors freed afterwards."""
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


# ---------------------------------------------------------------------------------------------------------------
# operands
# ---------------------------------------------------------------------------------------------------------------
def make_shard_case(W, N, C, Ks, variant, seed, skip=()):
    """(q, k, queue, plants) for W ranks of N queries and W shards of Ks rows.  plants = [(query i, queue row j)] with
    queue[j] == q[i]: shard r's t-th planted row takes a query of rank (r + 1 + t) % W, so every rank's queries are
    planted and, for W >= 2, each shard holds another rank's.  Queries in `skip` are never planted."""
    Nq, K = W * N, W * Ks
    rng = np.random.default_rng(seed)
    if variant == "tagged":
        q = exact_rows(rng, Nq, C, signed=False)
        k = np.zeros((Nq, C), np.float32)
        queue = tagged_rows(seed, K, C)
    else:
        q, k, queue = exact_rows(rng, Nq, C), exact_rows(rng, Nq, C), exact_rows(rng, K, C)
    plants = []
    for r in range(W):
        for t, p in enumerate(plant_positions(Ks, N)):
            i = ((r + 1 + t) % W) * N + (3 * t + r) % N
            while i in skip:
                i = (i + 1) % Nq
            plants.append((i, r * Ks + p))
            queue[r * Ks + p] = q[i]
    return q, k, queue, plants


# ---------------------------------------------------------------------------------------------------------------
# float64 per shard
# ---------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def shard_terms(q, queue, W, inv_T, lse, chunk=8192):
    """Per shard r, in float64 on the device: L[r] = log sum_{j in shard r} exp(x_ij) (natural log), and
    S[r] = sum_{j in shard r} p_ij m_j, A[r] = sum_{j in shard r} p_ij |m_j| with p_ij = exp(x_ij - lse_i)."""
    Nq, C = q.shape
    Ks = queue.shape[0] // W
    qd = torch.from_numpy(q).cuda().double()
    lse_d = torch.from_numpy(lse).cuda()
    L = np.empty((W, Nq))
    S = np.empty((W, Nq, C))
    A = np.empty((W, Nq, C))
    for r in range(W):
        l = torch.full((Nq,), -math.inf, dtype=torch.float64, device="cuda")
        s = torch.zeros(Nq, C, dtype=torch.float64, device="cuda")
        a = torch.zeros_like(s)
        for j0 in range(0, Ks, chunk):
            m = torch.from_numpy(queue[r * Ks + j0:r * Ks + min(j0 + chunk, Ks)]).cuda().double()
            x = qd @ m.T * inv_T
            l = torch.logaddexp(l, torch.logsumexp(x, 1))
            p = torch.exp(x - lse_d[:, None])
            s += p @ m
            a += p @ m.abs()
        L[r], S[r], A[r] = l.cpu().numpy(), s.cpu().numpy(), a.cpu().numpy()
    return L, S, A


def fma32(a, b, c):
    """fp32 fma(a, b, c) with one rounding: a * b is exact in float64, a * b + c is rounded to odd in float64 (TwoSum
    gives the exact error), and rounding that to fp32 is then the correctly rounded fused result."""
    a, b, c = np.broadcast_arrays(*(np.asarray(x, np.float32).astype(np.float64) for x in (a, b, c)))
    s = a * b
    t = np.ascontiguousarray(s + c)
    z = t - s
    e = (s - (t - z)) + (c - z)
    fix = (e != 0) & ((t.view(np.int64) & 1) == 0)
    t[fix] = np.nextafter(t[fix], np.where(e[fix] > 0, np.inf, -np.inf))
    return t.astype(np.float32)


def finish_restated(o_blocks, k_own, prob_own, N, inv_T):
    """The fp32 restatement of both finish kernels (module docstring): o summed in rank order from 0, then
    FMUL(FFMA(prob - 1, k, acc), inv_T / N)."""
    acc = np.zeros_like(o_blocks[0], dtype=np.float32)
    for o in o_blocks:
        acc = acc + o
    gscale = np.float32(np.float32(inv_T) / np.float32(N))
    pm1 = prob_own.astype(np.float32) - np.float32(1.0)
    return fma32(pm1[:, None], k_own, acc) * gscale


# ---------------------------------------------------------------------------------------------------------------
# running the chain
# ---------------------------------------------------------------------------------------------------------------
def _to_gpu(q, k, queue, W, dtype):
    tdt = torch.float32 if dtype == "f32" else torch.bfloat16
    Ks = queue.shape[0] // W
    shards = [torch.from_numpy(queue[r * Ks:(r + 1) * Ks]).cuda().bfloat16() for r in range(W)]
    return torch.from_numpy(q).cuda().to(tdt), torch.from_numpy(k).cuda().to(tdt), shards


def merge_on_fresh_workspace(qt, kt, shard0, ms_all, inv_T, flags):
    """Rank 0's statistics call and the merge again, on a workspace of their own: the pair must reproduce
    ms_all[0], and the merge gives loss_prob (simulate keeps each rank's own rows' means only)."""
    L = _lib()
    lib = L.load()
    s = L.cur_stream()
    W, Nq = ms_all.shape[:2]
    C, Ks = qt.shape[1], shard0.shape[0]
    ws, ptr, nbytes = _workspace(lib, Nq, C, Ks)
    f = dict(dtype=torch.float32, device="cuda")
    ms0 = torch.empty(Nq, 2, **f)
    L.check(lib.moco_nce_shard_stats(qt.data_ptr(), kt.data_ptr(), L.dtype_code(qt), shard0.data_ptr(), Nq, C, Ks, inv_T,
                                     ms0.data_ptr(), ptr, nbytes, flags, s), "moco_nce_shard_stats")
    out = {"lse": torch.empty(Nq, **f), "loss_rows": torch.empty(Nq, **f), "prob_rows": torch.empty(Nq, **f),
           "loss_prob": torch.empty(2, **f)}
    L.check(lib.moco_nce_shard_merge(ms_all.data_ptr(), W, Nq, C, inv_T, out["lse"].data_ptr(),
                                     out["loss_rows"].data_ptr(), out["prob_rows"].data_ptr(),
                                     out["loss_prob"].data_ptr(), ptr, nbytes, s), "moco_nce_shard_merge")
    torch.cuda.synchronize()
    return ms0, out


def chain_with_finish(qt, kt, shards, N, inv_T, flags):
    """The chain of simulate() for any world up to the merge's 160, finished with moco_nce_shard_dq_finish on the
    rank-order sum (moco_nce_shard_dq_finish_peers stops at 16)."""
    L = _lib()
    lib = L.load()
    s = L.cur_stream()
    W = len(shards)
    Nq, C = qt.shape
    Ks = shards[0].shape[0]
    dt = L.dtype_code(qt)
    f = dict(dtype=torch.float32, device="cuda")
    ws = [_workspace(lib, Nq, C, Ks) for _ in range(W)]
    ms = [torch.empty(Nq, 2, **f) for _ in range(W)]
    for r in range(W):
        L.check(lib.moco_nce_shard_stats(qt.data_ptr(), kt.data_ptr(), dt, shards[r].data_ptr(), Nq, C, Ks, inv_T,
                                         ms[r].data_ptr(), ws[r][1], ws[r][2], flags, s), "moco_nce_shard_stats")
    ms_all = torch.stack(ms)
    lse, loss_rows, prob_rows = ([torch.empty(Nq, **f) for _ in range(W)] for _ in range(3))
    loss_prob = [torch.empty(2, **f) for _ in range(W)]
    for r in range(W):
        L.check(lib.moco_nce_shard_merge(ms_all.data_ptr(), W, Nq, C, inv_T, lse[r].data_ptr(), loss_rows[r].data_ptr(),
                                         prob_rows[r].data_ptr(), loss_prob[r].data_ptr(), ws[r][1], ws[r][2], s),
                "moco_nce_shard_merge")
    o_part = [torch.empty(Nq, C, **f) for _ in range(W)]
    for r in range(W):
        L.check(lib.moco_nce_shard_dq(qt.data_ptr(), dt, shards[r].data_ptr(), lse[r].data_ptr(), Nq, C, Ks, inv_T,
                                      o_part[r].data_ptr(), ws[r][1], ws[r][2], flags, s), "moco_nce_shard_dq")
    dq_sum = []
    for r in range(W):
        own = slice(r * N, (r + 1) * N)
        o_own = o_part[0][own].clone()
        for rr in range(1, W):
            o_own += o_part[rr][own]
        d = torch.empty(N, C, **f)
        L.check(lib.moco_nce_shard_dq_finish(o_own.data_ptr(), kt[own].data_ptr(), dt, prob_rows[r][own].data_ptr(), N,
                                             C, inv_T, d.data_ptr(), s), "moco_nce_shard_dq_finish")
        dq_sum.append(d)
    torch.cuda.synchronize()
    return dict(ms_all=ms_all, lse=lse, loss_rows=loss_rows, prob_rows=prob_rows, loss_prob=loss_prob, o_part=o_part,
                dq_sum=dq_sum)


def run(case, W, N, dtype, flag, T):
    """simulate() for W <= 16 (plus rank 0's merge again, for loss_prob), chain_with_finish() beyond."""
    q, k, queue, _ = case
    inv_T = _fp32_inv_T(T)
    qt, kt, shards = _to_gpu(q, k, queue, W, dtype)
    if W > 16:
        out = chain_with_finish(qt, kt, shards, N, inv_T, FLAGS[flag])
        merged = {key: out[key][0] for key in ("lse", "loss_rows", "prob_rows", "loss_prob")}
        for r in range(1, W):
            assert torch.equal(out["loss_prob"][r], out["loss_prob"][0]), r
        return out, merged
    out = simulate(qt, kt, shards, N, T, FLAGS[flag])
    ms0, merged = merge_on_fresh_workspace(qt, kt, shards[0], out["ms_all"], inv_T, FLAGS[flag])
    assert torch.equal(ms0, out["ms_all"][0])
    for key in ("lse", "loss_rows", "prob_rows"):
        assert torch.equal(merged[key], out[key][0]), key
    return out, merged


# ---------------------------------------------------------------------------------------------------------------
# the four checks
# ---------------------------------------------------------------------------------------------------------------
def check_chain(case, out, merged, W, N, T, flag, unplanted=()):
    """Checks 1-4 of the module docstring.  `unplanted`: query rows (the power-of-two-norm rows) left out of the
    tagged variant's relative claim, whose partials on most shards are near fp32's underflow."""
    q, k, queue, plants = case
    inv_T = _fp32_inv_T(T)
    Nq, C = q.shape
    K = queue.shape[0]
    Ks = K // W
    tagged = not k.any()
    lse, loss_rows, prob_rows, S, A = reference(q, k, queue, inv_T)
    tol = lse_tol(lse)
    Ln, Sr, Ar = shard_terms(q, queue, W, inv_T, lse)
    assert (np.abs(Sr.sum(0) - S) <= 1e-9 * A).all()                            # the shards make up the queue

    # 1. each rank's (max, sum), log2 domain
    ms = out["ms_all"].cpu().numpy().astype(np.float64)
    assert ms.shape == (W, Nq, 2)
    with np.errstate(divide="ignore"):
        got = ms[..., 0] + np.log2(ms[..., 1])
    want = Ln / LN2
    tol2 = lse_tol(Ln) / LN2
    err = np.abs(got - want)
    assert np.isfinite(got).all() and (err <= tol2).all(), (float(np.nanmax(err / tol2)), np.argwhere(~(err <= tol2))[:5])
    for i, j in plants:                # one planted row more or less moves its shard's statistic past the tolerance
        r = j // Ks
        dup = math.log1p(math.exp(inv_T - Ln[r, i])) / LN2
        assert dup > tol2[r, i], (r, i, j, dup, tol2[r, i])
    if flag == "one_pass":             # the sweep's constant stabiliser, or the exact pair (lse2, 1)
        stab = np.float32(inv_T) * np.float32(1.4426950408889634)
        assert ((ms[..., 0] == stab) | (ms[..., 1] == 1.0)).all()

    # 2. the merge
    for r in range(1, W):
        for key in ("lse", "loss_rows", "prob_rows"):
            assert torch.equal(out[key][r], out[key][0]), (key, r)
    assert_planted_rows_matter(lse, inv_T, plants, tol)
    check_stats(merged, lse, loss_rows, prob_rows, tol)

    # 3. each rank's o_partial
    zero_k = np.zeros_like(q)
    keep = np.ones(Nq, bool)
    keep[list(unplanted)] = False
    for r in range(W):
        o = out["o_part"][r].cpu().numpy().astype(np.float64)
        exp, bound = dq_expected_and_bound(zero_k, 1.0, 1, Ks, prob_rows, tol, Sr[r], Ar[r])
        bad = ~(np.abs(o - exp) <= bound)
        assert not bad.any(), (r, int(bad.sum()), np.argwhere(bad)[:5].tolist())
        if tagged:
            nz = (exp > 0) & keep[:, None]
            assert (bound[nz] / exp[nz]).max() < BF16_P + gamma(Ks + 8) + 2 * tol.max() + 1e-4
            for i, j in [p for p in plants if p[1] // Ks == r][:64]:
                share = np.exp(inv_T - lse[i]) * queue[j].astype(np.float64)
                c = int(np.argmax(share))
                assert share[c] > 2 * bound[i, c], (r, i, j, share[c] / bound[i, c])

    # 4. the finish: both kernels, bit for bit against the restatement, then against float64
    o_parts = [t.cpu().numpy() for t in out["o_part"]]
    for r in range(W):
        own = slice(r * N, (r + 1) * N)
        prob_own = out["prob_rows"][r][own].cpu().numpy()
        want = finish_restated([o[own] for o in o_parts], k[own], prob_own, N, inv_T)
        got = out["dq_sum"][r].cpu().numpy()
        np.testing.assert_array_equal(got, want)
        if "dq_peers" in out:
            np.testing.assert_array_equal(out["dq_peers"][r].cpu().numpy(), got)
        exp, bound = dq_expected_and_bound(k[own], inv_T, N, K, prob_rows[own], tol[own], S[own], A[own])
        bad = ~(np.abs(got.astype(np.float64) - exp) <= bound)
        assert not bad.any(), (r, int(bad.sum()), np.argwhere(bad)[:5].tolist())


# ---------------------------------------------------------------------------------------------------------------
# the matrix: a sampled product
# ---------------------------------------------------------------------------------------------------------------
MATRIX = [  # (W, Ks, N per rank, C, q/k dtype, flag, T, variant)
    (1, 1, 1, 64, "f32", "one_pass", 0.07, "signed"),
    (2, 63, 37, 128, "bf16", "two_pass", 0.07, "tagged"),
    (3, 64, 256, 192, "f32", "cta_pair", 0.03, "signed"),
    (5, 65, 37, 256, "bf16", "one_pass", 0.07, "tagged"),
    (8, 127, 1, 64, "f32", "two_pass", 0.03, "tagged"),
    (16, 128, 37, 128, "bf16", "cta_pair", 0.07, "signed"),
    (2, 129, 256, 64, "f32", "one_pass", 0.03, "signed"),
    (3, 4096 + 77, 37, 128, "f32", "one_pass", 0.07, "tagged"),
    (5, 16384, 1, 192, "bf16", "two_pass", 0.07, "signed"),
    (8, 16384, 37, 64, "f32", "one_pass", 0.07, "tagged"),             # 8 x 16384 rows: BASELINE configs[3]
    (16, 16384, 1, 128, "bf16", "two_pass", 0.03, "tagged"),
    (2, 16384, 256, 256, "f32", "cta_pair", 0.07, "signed"),
    (3, 16384, 37, 256, "f32", "two_pass", 0.03, "signed"),
    (5, 4096 + 77, 256, 64, "bf16", "cta_pair", 0.03, "tagged"),
    (16, 65, 256, 192, "f32", "two_pass", 0.07, "signed"),
    (1, 16384, 256, 128, "bf16", "one_pass", 0.03, "tagged"),           # forced one sweep at 1/T > 25
    (2, 4096 + 77, 1, 256, "bf16", "cta_pair", 0.03, "signed"),
    (16, 1, 37, 256, "f32", "one_pass", 0.07, "tagged"),
    (8, 63, 256, 128, "f32", "cta_pair", 0.07, "tagged"),
    (5, 128, 1, 128, "f32", "one_pass", 0.03, "signed"),
    (3, 129, 37, 64, "bf16", "two_pass", 0.07, "tagged"),
    (1, 127, 37, 256, "bf16", "cta_pair", 0.03, "signed"),
]


def _id(c):
    return f"W{c[0]}-Ks{c[1]}-N{c[2]}-C{c[3]}-{c[4]}-{c[5]}-T{c[6]}-{c[7]}"


@pytest.mark.parametrize("W,Ks,N,C,dtype,flag,T,variant", MATRIX, ids=[_id(c) for c in MATRIX])
def test_shard_chain_link_by_link(W, Ks, N, C, dtype, flag, T, variant):
    case = make_shard_case(W, N, C, Ks, variant, seed=W * 7919 + Ks * 31 + N * 7 + C)
    out, merged = run(case, W, N, dtype, flag, T)
    check_chain(case, out, merged, W, N, T, flag)


def test_matrix_covers_every_world_shard_flag_dtype_and_temperature():
    """The sampled product runs every W, Ks, N, C, dtype, flag, temperature and variant at least once."""
    assert {m[0] for m in MATRIX} == {1, 2, 3, 5, 8, 16}
    assert {m[1] for m in MATRIX} == {1, 63, 64, 65, 127, 128, 129, 4096 + 77, 16384}
    assert {m[2] for m in MATRIX} == {1, 37, 256}
    assert {m[3] for m in MATRIX} == {64, 128, 192, 256}
    assert {m[4] for m in MATRIX} == {"f32", "bf16"}
    assert {m[5] for m in MATRIX} == set(FLAGS)
    assert {m[6] for m in MATRIX} == {0.07, 0.03}
    assert {m[7] for m in MATRIX} == {"tagged", "signed"}


# ---------------------------------------------------------------------------------------------------------------
# the merge alone at large worlds
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W,Ks,C,dtype,flag,T", [(33, 3, 128, "bf16", "one_pass", 0.07),
                                                 (160, 2, 64, "f32", "two_pass", 0.03)])
def test_merge_at_large_worlds(W, Ks, C, dtype, flag, T):
    """world = 33 and 160 (the merge's maximum) with one query per rank and a tiny shard each."""
    case = make_shard_case(W, 1, C, Ks, "signed", seed=W + Ks)
    out, merged = run(case, W, 1, dtype, flag, T)
    check_chain(case, out, merged, W, 1, T, flag)


# ---------------------------------------------------------------------------------------------------------------
# one-sweep rows that need the exact evaluation on one shard only
# ---------------------------------------------------------------------------------------------------------------
def plant_fallback_rows(case, W, N, Ks, T, rows):
    """Scale each q row in `rows` to a power-of-two norm s and put a partner row v (o of q's 16 entries, 16 - o
    elsewhere) in shard (rank + 1) % W only: <q, v> = s o / 16 is exact and lands 102-114 binades above the one-sweep
    stabiliser, past its 2^100 slice limit, while the merge weight 2^(stabiliser - lse2) of the other shards stays a
    normal fp32 number.  Returns {row: shard holding its partner}."""
    q, k, queue, plants = case
    C = q.shape[1]
    inv_T = _fp32_inv_T(T)
    stab = inv_T / LN2
    choice = next((s, o) for s in (4.0, 8.0, 16.0) for o in range(1, 17) if 102 <= s * o / 16 * stab - stab <= 114)
    s, o = choice
    taken = {j for _, j in plants}
    where = {}
    for n, i in enumerate(rows):
        u = q[i].copy()
        support = np.flatnonzero(u)
        v = np.zeros(C, np.float32)
        v[support[:o]] = u[support[:o]]
        outside = np.setdiff1d(np.arange(C), support)[n:n + 16 - o]
        v[outside] = 0.25
        q[i] = u * s
        r = (i // N + 1) % W
        j = r * Ks + Ks // 2
        while j in taken:
            j += 1
        assert j < (r + 1) * Ks
        taken.add(j)
        queue[j] = v
        where[i] = r
    return where


@pytest.mark.parametrize("W,Ks,N,C,dtype,T,variant", [(3, 4096 + 77, 37, 128, "f32", 0.07, "signed"),
                                                      (2, 129, 37, 64, "bf16", 0.03, "tagged"),
                                                      (5, 65, 37, 256, "f32", 0.07, "tagged"),
                                                      (8, 16384, 1, 192, "bf16", 0.03, "signed")])
def test_exact_rows_on_one_shard_only(W, Ks, N, C, dtype, T, variant):
    rows = sorted({N // 2, (W - 1) * N + N - 1})
    case = make_shard_case(W, N, C, Ks, variant, seed=W * 13 + Ks + C, skip=set(rows))
    where = plant_fallback_rows(case, W, N, Ks, T, rows)
    q, k, queue, _ = case
    inv_T = _fp32_inv_T(T)
    # float64: the partner's term alone is past 2^100 on its shard; every other shard sums to well inside the range
    stab = inv_T / LN2
    lse, *_ = reference(q, k, queue, inv_T)
    Ln, _, _ = shard_terms(q, queue, W, inv_T, lse)
    qd = q[rows].astype(np.float64)
    for n, i in enumerate(rows):
        for r in range(W):
            top = (qd[n] @ queue[r * Ks:(r + 1) * Ks].astype(np.float64).T).max() * inv_T / LN2 - stab
            if r == where[i]:
                assert top > 101, (i, r, top)
            else:
                assert -79 < Ln[r, i] / LN2 - stab < 99, (i, r, Ln[r, i] / LN2 - stab)
    out, merged = run(case, W, N, dtype, "one_pass", T)
    ms = out["ms_all"].cpu().numpy()
    stab32 = np.float32(inv_T) * np.float32(1.4426950408889634)
    for i in rows:                     # the exact pair where the partner is, the sweep's pair everywhere else
        for r in range(W):
            if r == where[i]:
                assert ms[r, i, 1] == 1.0 and ms[r, i, 0] > stab32 + 100, (i, r, ms[r, i])
            else:
                assert ms[r, i, 0] == stab32, (i, r, ms[r, i])
    check_chain(case, out, merged, W, N, T, "one_pass", unplanted=rows)


# ---------------------------------------------------------------------------------------------------------------
# the envelope's edge
# ---------------------------------------------------------------------------------------------------------------
def largest_nq(flag, sms):
    """The statistics kernels' rule, mblks * G <= #SM with mblks = ceil(Nq / (128 G)) (G = 2 for the CTA pair): the
    one-sweep and dq sweeps take mblks = ceil(Nq / 128) <= #SM, which is never smaller."""
    G = 2 if flag == "cta_pair" else 1
    return 128 * G * (sms // G)


@pytest.mark.parametrize("flag", list(FLAGS))
def test_envelope_edge(flag):
    """At the largest Nq the tensor-core statistics accept, the whole chain is exact; one row more is refused with
    MOCO_ERR_UNSUPPORTED and a message, by the statistics and by the dq call."""
    W, Ks, C, T = 2, 65, 64, 0.07
    nq = largest_nq(flag, _sms())
    case = make_shard_case(W, nq // W, C, Ks, "signed", seed=nq)
    out, merged = run(case, W, nq // W, "bf16", flag, T)
    check_chain(case, out, merged, W, nq // W, T, flag)
    del out, merged

    L = _lib()
    lib = L.load()
    s = L.cur_stream()
    n1 = nq + 1
    rng = np.random.default_rng(n1)
    qt = torch.from_numpy(exact_rows(rng, n1, C)).cuda().bfloat16()
    shard = torch.from_numpy(exact_rows(rng, Ks, C)).cuda().bfloat16()
    ws, ptr, nbytes = _workspace(lib, n1, C, Ks)
    f = dict(dtype=torch.float32, device="cuda")
    ms = torch.full((n1, 2), float("nan"), **f)
    lse = torch.zeros(n1, **f)
    o = torch.full((n1, C), float("nan"), **f)
    rc = lib.moco_nce_shard_stats(qt.data_ptr(), qt.data_ptr(), L.dtype_code(qt), shard.data_ptr(), n1, C, Ks,
                                  _fp32_inv_T(T), ms.data_ptr(), ptr, nbytes, FLAGS[flag], s)
    msg = lib.moco_last_error().decode()
    assert rc == MOCO_ERR_UNSUPPORTED and "not supported" in msg, (rc, msg)
    rc = lib.moco_nce_shard_dq(qt.data_ptr(), L.dtype_code(qt), shard.data_ptr(), lse.data_ptr(), n1, C, Ks,
                               _fp32_inv_T(T), o.data_ptr(), ptr, nbytes, FLAGS[flag], s)
    msg = lib.moco_last_error().decode()
    assert rc == MOCO_ERR_UNSUPPORTED and "not supported" in msg, (rc, msg)
    torch.cuda.synchronize()
    assert bool(torch.isnan(ms).all()) and bool(torch.isnan(o).all())      # nothing was written
