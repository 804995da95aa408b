"""The sharded-queue head (moco_nce_shard_stats / _merge / _dq / _dq_finish / _dq_finish_peers, include/moco_b200.h) at
2-16 simulated ranks on one GPU.  Every entry point takes raw device pointers, so W ranks are W sets of buffers on the
same device: W shards, W workspaces, the W (max, sum) outputs stacked as the all_gather would stack them, and the W
o_partial buffers handed to _dq_finish_peers as its peer table.  The call sequence is ShardedContrast._ShardedNCE's.

The reference is the replicated head over the whole queue (the loss is permutation-invariant over negatives), in
float64, with the kernels' operand contract: negatives <bf16(q), queue_j> / T, the positive <q, k> / T from the inputs
as given, and rank r's dq the gradient of the mean over its own N rows."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import moco_oracle as O
from tests.helpers import rand_unit

pytestmark = pytest.mark.gpu

LSE_ATOL = 2e-4
DQ_RTOL = 5e-3          # of max|dq|: P is rounded to bf16 before the P.Queue MMA


def _lib():
    from moco_b200 import _lib
    return _lib


def _workspace(lib, Nq, C, Ks):
    n = int(lib.moco_nce_workspace_bytes(Nq, C, Ks))
    t = torch.empty(n + 256, dtype=torch.uint8, device="cuda")
    return t, t.data_ptr() + (-t.data_ptr()) % 256, n


def simulate(q_all, k_all, shards, N, T, flags):
    """One head step of W = len(shards) ranks, rank r holding shards[r] ([Ks, C] bf16) and queries
    [r*N, (r+1)*N) of q_all / k_all ([W*N, C], fp32 or bf16)."""
    L = _lib()
    lib = L.load()
    s = L.cur_stream()
    W = len(shards)
    Nq, C = q_all.shape
    Ks = shards[0].shape[0]
    inv_T = 1.0 / T
    dt = L.dtype_code(q_all)
    f32 = dict(dtype=torch.float32, device="cuda")
    ws = [_workspace(lib, Nq, C, Ks) for _ in range(W)]
    ms = [torch.empty(Nq, 2, **f32) for _ in range(W)]
    for r in range(W):
        L.check(lib.moco_nce_shard_stats(q_all.data_ptr(), k_all.data_ptr(), dt, shards[r].data_ptr(), Nq, C, Ks, inv_T,
                                         ms[r].data_ptr(), ws[r][1], ws[r][2], flags, s), "moco_nce_shard_stats")
    ms_all = torch.stack(ms)                                           # the all_gather: [W, Nq, 2]
    lse, loss_rows, prob_rows = ([torch.empty(Nq, **f32) for _ in range(W)] for _ in range(3))
    loss_prob = [torch.empty(2, **f32) for _ in range(W)]
    for r in range(W):
        L.check(lib.moco_nce_shard_merge(ms_all.data_ptr(), W, Nq, C, inv_T, lse[r].data_ptr(), loss_rows[r].data_ptr(),
                                         prob_rows[r].data_ptr(), loss_prob[r].data_ptr(), ws[r][1], ws[r][2], s),
                "moco_nce_shard_merge")
    o_part = [torch.empty(Nq, C, **f32) for _ in range(W)]
    for r in range(W):
        L.check(lib.moco_nce_shard_dq(q_all.data_ptr(), dt, shards[r].data_ptr(), lse[r].data_ptr(), Nq, C, Ks, inv_T,
                                      o_part[r].data_ptr(), ws[r][1], ws[r][2], flags, s), "moco_nce_shard_dq")
    peers = (ctypes.c_void_p * W)(*[o.data_ptr() for o in o_part])
    dq_peers, dq_sum, loss, prob = [], [], [], []
    for r in range(W):
        own = slice(r * N, (r + 1) * N)
        k_own, prob_own = k_all[own], prob_rows[r][own]
        d = torch.empty(N, C, **f32)
        L.check(lib.moco_nce_shard_dq_finish_peers(peers, W, r, k_own.data_ptr(), dt, prob_own.data_ptr(), N, C, inv_T,
                                                   d.data_ptr(), s), "moco_nce_shard_dq_finish_peers")
        dq_peers.append(d)
        o_own = o_part[0][own].clone()                                 # the reduce_scatter, summed in rank order
        for rr in range(1, W):
            o_own += o_part[rr][own]
        d = torch.empty(N, C, **f32)
        L.check(lib.moco_nce_shard_dq_finish(o_own.data_ptr(), k_own.data_ptr(), dt, prob_own.data_ptr(), N, C, inv_T,
                                             d.data_ptr(), s), "moco_nce_shard_dq_finish")
        dq_sum.append(d)
        loss.append(float(loss_rows[r][own].mean()))                   # this rank's loss and prob: its own rows
        prob.append(float(prob_rows[r][own].mean()))
    torch.cuda.synchronize()
    return dict(ms_all=ms_all, lse=lse, loss_rows=loss_rows, prob_rows=prob_rows, o_part=o_part,
                dq_peers=dq_peers, dq_sum=dq_sum, loss=loss, prob=prob)


@torch.no_grad()
def reference(q_all, k_all, queue, N, T, chunk=8192):
    """float64 head over the whole queue: (lse, loss_rows, prob_rows, dq) for all W*N rows."""
    qb = q_all.to(torch.bfloat16).double()                             # the MMA operand: bf16(q)
    q64, k64, mem = q_all.double(), k_all.double(), queue.double()
    x0 = (q64 * k64).sum(1) / T
    lse = x0.clone()
    for j0 in range(0, mem.shape[0], chunk):
        lse = torch.logaddexp(lse, torch.logsumexp(qb @ mem[j0:j0 + chunk].T / T, 1))
    p0 = torch.exp(x0 - lse)
    acc = (p0 - 1.0)[:, None] * k64
    for j0 in range(0, mem.shape[0], chunk):
        m = mem[j0:j0 + chunk]
        acc += torch.exp(qb @ m.T / T - lse[:, None]) @ m
    return lse, lse - x0, p0, acc / (T * N)


def _inputs(rng, W, N, C, Ks, q_scale=1.0):
    Nq, K = W * N, W * Ks
    q, k, mem = rand_unit(rng, Nq, C), rand_unit(rng, Nq, C), rand_unit(rng, K, C)
    if q_scale != 1.0:
        q = O.bf16_round(q * q_scale)
    return q, k, mem


def _to_gpu(q, k, mem, W, dtype):
    qt = torch.from_numpy(q).cuda().to(dtype)
    kt = torch.from_numpy(k).cuda().to(dtype)
    queue = torch.from_numpy(mem).cuda().bfloat16()
    Ks = queue.shape[0] // W
    shards = [queue[r * Ks:(r + 1) * Ks].clone() for r in range(W)]
    return qt, kt, queue, shards


def _check_vs_reference(out, ref, W, N):
    lse_ref, loss_rows_ref, prob_rows_ref, dq_ref = ref
    for r in range(W):
        own = slice(r * N, (r + 1) * N)
        lse_err = float((out["lse"][r].double() - lse_ref).abs().max())
        assert lse_err < LSE_ATOL, (r, lse_err)
        loss = float(loss_rows_ref[own].mean())
        prob = float(prob_rows_ref[own].mean())
        assert np.isfinite(out["loss"][r]) and abs(out["loss"][r] - loss) < 2e-4 * max(1.0, abs(loss)), (r, out["loss"][r], loss)
        assert abs(out["prob"][r] - prob) < 1e-3 * prob + 1e-9, (r, out["prob"][r], prob)
    dq = torch.cat(out["dq_peers"]).double()
    assert bool(torch.isfinite(dq).all())
    dq_err = float((dq - dq_ref).abs().max() / dq_ref.abs().max())
    assert dq_err < DQ_RTOL, dq_err


def _check_consistency(out, W):
    """Every rank merges the same [W, Nq] pairs: bit-identical lse / loss_rows / prob_rows; the two finish kernels
    agree."""
    for r in range(1, W):
        for key in ("lse", "loss_rows", "prob_rows"):
            assert torch.equal(out[key][r], out[key][0]), (key, r)
    for a, b in zip(out["dq_peers"], out["dq_sum"]):
        torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-6 * float(b.abs().max()))


def _flag(name):
    L = _lib()
    return {"one_pass": L.NCE_ONE_PASS, "two_pass": 0, "cta_pair": L.NCE_CTA_PAIR}[name]


# (W, C, N per rank, Ks, q/k dtype, flags, T): 15 points of the product, each W, C, N, Ks, dtype, flag and T appearing
# several times; 16384 rows per rank at W = 8 is BASELINE configs[3].
CASES = [
    (2, 128, 37, 4096 + 77, "f32", "one_pass", 0.07),
    (4, 64, 1, 50, "bf16", "one_pass", 0.07),
    (8, 128, 256, 16384, "f32", "one_pass", 0.07),
    (16, 256, 37, 4096 + 77, "f32", "one_pass", 0.07),
    (4, 192, 256, 50, "f32", "one_pass", 0.07),
    (2, 192, 37, 50, "bf16", "one_pass", 0.07),
    (2, 256, 1, 16384, "bf16", "two_pass", 0.07),
    (8, 64, 37, 4096 + 77, "f32", "two_pass", 0.07),
    (16, 128, 1, 50, "bf16", "two_pass", 0.07),
    (4, 128, 256, 4096 + 77, "bf16", "cta_pair", 0.07),
    (8, 192, 37, 16384, "f32", "cta_pair", 0.07),
    (2, 64, 256, 16384, "f32", "cta_pair", 0.07),
    (4, 128, 37, 4096 + 77, "f32", "one_pass", 0.03),      # forced one sweep at 1/T > 25: exact for unit-norm rows
    (16, 64, 256, 50, "bf16", "one_pass", 0.03),
    (8, 256, 1, 4096 + 77, "bf16", "two_pass", 0.03),
]


@pytest.mark.parametrize("W,C,N,Ks,dtype,flag,T", CASES,
                         ids=[f"W{c[0]}-C{c[1]}-N{c[2]}-Ks{c[3]}-{c[4]}-{c[5]}-T{c[6]}" for c in CASES])
def test_simulated_ranks_match_reference(W, C, N, Ks, dtype, flag, T):
    rng = np.random.default_rng(W * 1000 + C + N + Ks)
    dtype = torch.float32 if dtype == "f32" else torch.bfloat16
    q, k, mem = _inputs(rng, W, N, C, Ks)
    qt, kt, queue, shards = _to_gpu(q, k, mem, W, dtype)
    out = simulate(qt, kt, shards, N, T, _flag(flag))
    _check_vs_reference(out, reference(qt, kt, queue, N, T), W, N)
    _check_consistency(out, W)
    again = simulate(qt, kt, shards, N, T, _flag(flag))                # the whole step is deterministic
    for key in ("ms_all", "lse", "loss_rows", "prob_rows", "dq_peers", "dq_sum"):
        a, b = out[key], again[key]
        for x, y in (zip(a, b) if isinstance(a, list) else [(a, b)]):
            assert torch.equal(x, y), key


@pytest.mark.parametrize("flag", ["one_pass", "two_pass", "cta_pair"])
def test_uneven_shards_rescale_in_the_merge(flag):
    """Queries whose own direction (logit +1/T) sits in shard 1 and whose negation (-1/T) sits in the ragged last tile
    of shard 3: shard 1's maximum of those rows is the largest logit there can be, far above shard 3's, so the merge
    must rescale the shards' sums against each other."""
    W, C, N, Ks, T = 4, 128, 37, 4096 + 77, 0.07
    rng = np.random.default_rng(5)
    q, k, mem = _inputs(rng, W, N, C, Ks)
    rows = [0, 3, 40, 77, 100, 147]                                    # queries of every rank
    for n, i in enumerate(rows):
        mem[1 * Ks + 500 + 7 * n] = q[i]                               # logit +1/T
        mem[3 * Ks + Ks - 1 - 5 * n] = -q[i]                           # logit -1/T, in the ragged last tile
    qt, kt, queue, shards = _to_gpu(q, k, mem, W, torch.float32)
    out = simulate(qt, kt, shards, N, T, _flag(flag))
    if flag != "one_pass":                                             # the statistics kernel's running maxima, log2 domain
        ms = out["ms_all"].cpu().numpy().astype(np.float64)
        top = (q[rows].astype(np.float64) ** 2).sum(1) * np.log2(np.e) / T
        np.testing.assert_allclose(ms[1, rows, 0], top, atol=1e-3)
        assert np.all(ms[1, rows, 0] - ms[3, rows, 0] > 0.5 * np.log2(np.e) / T), ms[:, rows, 0]
    _check_vs_reference(out, reference(qt, kt, queue, N, T), W, N)
    _check_consistency(out, W)


@pytest.mark.parametrize("W", [1, 4])
@pytest.mark.parametrize("C", [128, 256])
def test_unnormalised_queries_one_sweep_stays_exact(C, W):
    """q of norm 12 with one row's exact direction in the last tile of the last shard: that logit is ~11/T nats
    (~226 binades at T = 0.07) above the one-sweep kernel's constant stabiliser, so its shard sum overflows.  Such rows
    are evaluated exactly on CUDA cores, and the head stays finite and equal to the reference."""
    N, Ks, T = 64 // W, 4096 + 77, 0.07
    rng = np.random.default_rng(C + W)
    q, k, mem = _inputs(rng, W, N, C, Ks, q_scale=12.0)
    mem[W * Ks - 7] = O.bf16_round(q[3] / 12.0)
    qt, kt, queue, shards = _to_gpu(q, k, mem, W, torch.float32)
    out = simulate(qt, kt, shards, N, T, _flag("one_pass"))
    _check_vs_reference(out, reference(qt, kt, queue, N, T), W, N)
    _check_consistency(out, W)


@pytest.mark.parametrize("C", [128, 256])
def test_unnormalised_queries_through_sharded_module(C):
    """The same inputs through ShardedMemoryMoCo at world 1 with its default flags (one sweep at T = 0.07 when a
    gradient is wanted) and through MemoryMoCo: the same loss, prob and dq, and both equal to the reference."""
    from moco_b200.NCE import MemoryMoCo, ShardedMemoryMoCo
    N, K, T = 64, 4096 + 77, 0.07
    rng = np.random.default_rng(C)
    q, k, mem = _inputs(rng, 1, N, C, K, q_scale=12.0)
    mem[K - 7] = O.bf16_round(q[3] / 12.0)
    results = []
    for cls in (ShardedMemoryMoCo, MemoryMoCo):
        mod = cls(C, K, T)
        mod.memory.copy_(torch.from_numpy(mem))
        mod = mod.cuda()
        qt = torch.from_numpy(q).cuda().requires_grad_(True)
        kt = torch.from_numpy(k).cuda()
        loss, prob = mod.forward_loss(qt, kt, kt)
        loss.backward()
        results.append((float(loss.detach()), float(prob), qt.grad.double()))
    qt, kt = torch.from_numpy(q).cuda(), torch.from_numpy(k).cuda()
    lse_ref, loss_rows_ref, prob_rows_ref, dq_ref = reference(qt, kt, torch.from_numpy(mem).cuda().bfloat16(), N, T)
    loss_ref, prob_ref = float(loss_rows_ref.mean()), float(prob_rows_ref.mean())
    for loss, prob, dq in results:
        assert np.isfinite(loss) and abs(loss - loss_ref) < 2e-4 * max(1.0, abs(loss_ref)), (loss, loss_ref)
        assert abs(prob - prob_ref) < 1e-3 * prob_ref + 1e-9, (prob, prob_ref)
        assert bool(torch.isfinite(dq).all()) and float((dq - dq_ref).abs().max() / dq_ref.abs().max()) < DQ_RTOL
    (ls, ps, gs), (lm, pm, gm) = results
    assert abs(ls - lm) < 2e-4 * max(1.0, abs(lm)) and abs(ps - pm) < 1e-3 * pm + 1e-9
    assert float((gs - gm).abs().max() / gm.abs().max()) < DQ_RTOL


@pytest.mark.parametrize("flag", ["one_pass", "two_pass"])
def test_three_steps_with_enqueue_across_the_ring_end(flag):
    """Three steps of W = 4 simulated ranks, each followed by moco_queue_enqueue_shard on every shard.  The ring
    position starts at K - 40, so the first write wraps from the last shard into the first.  Each step's loss and dq
    match the reference on the pre-enqueue queue; the reassembled queue matches the oracle's bit for bit."""
    L = _lib()
    lib = L.load()
    W, C, N, Ks, T = 4, 128, 37, 1024 + 13, 0.07
    K, Nq = W * Ks, W * N
    rng = np.random.default_rng(17)
    mem = rand_unit(rng, K, C)
    index = K - 40
    orc = O.MemoryMoCoOracle(mem, T, index=index)
    shards_f = [torch.from_numpy(mem[r * Ks:(r + 1) * Ks].copy()).cuda() for r in range(W)]
    shards_b = [s.bfloat16() for s in shards_f]
    for _ in range(3):
        q, k = rand_unit(rng, Nq, C), rand_unit(rng, Nq, C)
        qt, kt = torch.from_numpy(q).cuda(), torch.from_numpy(k).cuda()
        queue = torch.cat(shards_b)
        np.testing.assert_array_equal(queue.float().cpu().numpy(), O.bf16_round(orc.memory))
        out = simulate(qt, kt, shards_b, N, T, _flag(flag))
        _check_vs_reference(out, reference(qt, kt, queue, N, T), W, N)
        _check_consistency(out, W)
        orc.enqueue(k)
        for r in range(W):
            L.check(lib.moco_queue_enqueue_shard(shards_b[r].data_ptr(), shards_f[r].data_ptr(), kt.data_ptr(), L.MOCO_F32,
                                                 Nq, C, K, index, r * Ks, Ks, L.cur_stream()), "moco_queue_enqueue_shard")
        index = (index + Nq) % K
        assert index == orc.index
    np.testing.assert_array_equal(torch.cat(shards_f).cpu().numpy(), orc.memory)
    np.testing.assert_array_equal(torch.cat(shards_b).float().cpu().numpy(), O.bf16_round(orc.memory))
