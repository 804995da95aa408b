"""CPU oracle for the MoCo contrastive hot path (TEST INFRASTRUCTURE ONLY).

This file restates, in plain numpy, the algorithm of the reference's hot path
(bl0/moco).  Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs may import it.  The product
(``moco_b200``) never imports anything from ``oracle/``.

Parity pinning: the reference ships no tests, golden vectors or known-answer
files (SURVEY.md §4/§8c).  The oracle is therefore pinned against OUTPUTS OF
THE REFERENCE ITSELF: ``tests/golden/gen_golden.py`` imports the unmodified
reference from ``/root/reference`` (with the CPU shims described there), runs
it on seeded inputs and commits the results under ``tests/golden/*.npz``;
``tests/test_oracle_golden.py`` checks every function below against those
fixtures.  The arithmetic the reference delegates to PyTorch (third-party,
``pytorch>=1.3``, reference ``README.md:14``; 2.11.0 installed here) is restated
from its published algorithms: ``torch.randperm`` on the CPU generator is
MT19937 + a forward Fisher-Yates (`randperm_cpu`), ``nn.CrossEntropyLoss`` is
mean(logsumexp - x[label]).

Every function cites the reference file:line it follows (paths relative to
``/root/reference``).
"""
from __future__ import annotations

import math
from typing import List, Sequence, Tuple

import numpy as np

# --------------------------------------------------------------------------
# torch CPU generator restatement (MT19937) -- used by get_shuffle_ids
# --------------------------------------------------------------------------


class MT19937:
    """32-bit Mersenne Twister, `init_genrand(seed)` seeding.

    ``torch.manual_seed(s)`` seeds the CPU generator's mt19937 engine with
    ``s`` (low 32 bits) and ``generator->random()`` returns successive 32-bit
    outputs; this is the textbook MT19937 (Matsumoto & Nishimura 1998).
    """

    N, M = 624, 397

    def __init__(self, seed: int):
        mt = np.zeros(self.N, dtype=np.uint64)
        mt[0] = seed & 0xFFFFFFFF
        for i in range(1, self.N):
            prev = int(mt[i - 1])
            mt[i] = (1812433253 * (prev ^ (prev >> 30)) + i) & 0xFFFFFFFF
        self.mt = mt.astype(np.uint32)
        self.pos = self.N

    def _twist(self) -> None:
        mt = self.mt.astype(np.uint64)
        N, M = self.N, self.M
        # the recurrence reads already-updated words for i >= N-M, so do it in
        # three dependent vector blocks exactly like the scalar loop would.
        def blk(lo, hi, src_off):
            y = (mt[lo:hi] & 0x80000000) | (mt[lo + 1:hi + 1] & 0x7FFFFFFF)
            mag = np.where(y & 1, np.uint64(0x9908B0DF), np.uint64(0))
            mt[lo:hi] = mt[lo + src_off:hi + src_off] ^ (y >> np.uint64(1)) ^ mag
        blk(0, N - M, M)                     # i in [0, 227): uses mt[i+397] (old)
        blk(N - M, 2 * (N - M), M - N)       # i in [227, 454): uses mt[i-227] (new)
        blk(2 * (N - M), N - 1, M - N)       # i in [454, 623): uses mt[i-227] (new)
        y = (mt[N - 1] & 0x80000000) | (mt[0] & 0x7FFFFFFF)
        mag = np.uint64(0x9908B0DF) if (int(y) & 1) else np.uint64(0)
        mt[N - 1] = mt[M - 1] ^ (y >> np.uint64(1)) ^ mag
        self.mt = mt.astype(np.uint32)
        self.pos = 0

    def random_raw(self, n: int) -> np.ndarray:
        out = np.empty(n, dtype=np.uint32)
        got = 0
        while got < n:
            if self.pos >= self.N:
                self._twist()
            take = min(n - got, self.N - self.pos)
            y = self.mt[self.pos:self.pos + take].astype(np.uint64)
            y ^= y >> np.uint64(11)
            y ^= (y << np.uint64(7)) & np.uint64(0x9D2C5680)
            y ^= (y << np.uint64(15)) & np.uint64(0xEFC60000)
            y ^= y >> np.uint64(18)
            out[got:got + take] = (y & np.uint64(0xFFFFFFFF)).astype(np.uint32)
            self.pos += take
            got += take
        return out


def torch_cpu_randperm(n: int, seed: int) -> np.ndarray:
    """``torch.manual_seed(seed); torch.randperm(n)`` on the CPU generator.

    PyTorch's ``randperm_cpu`` (aten/src/ATen/native/TensorFactories.cpp):
    ``for i in [0, n-1): z = random() % (n-i); swap(r[i], r[i+z])``.
    Called by the reference at moco/util.py:102-104.
    """
    r = np.arange(n, dtype=np.int64)
    if n <= 1:
        return r
    raw = MT19937(seed).random_raw(n - 1)
    for i in range(n - 1):
        z = int(raw[i]) % (n - i)
        r[i], r[i + z] = r[i + z], r[i]
    return r


# --------------------------------------------------------------------------
# ShuffleBN  (reference moco/util.py:47-111)
# --------------------------------------------------------------------------


def get_shuffle_ids(bsz: int, epoch: int) -> Tuple[np.ndarray, np.ndarray]:
    """moco/util.py:99-111 -- forward permutation and its inverse (int64)."""
    forward_inds = torch_cpu_randperm(bsz, epoch)
    backward_inds = np.zeros(bsz, dtype=np.int64)
    backward_inds[forward_inds] = np.arange(bsz, dtype=np.int64)  # index_copy_, util.py:107-109
    return forward_inds, backward_inds


def dist_collect(xs: Sequence[np.ndarray]) -> np.ndarray:
    """moco/util.py:47-58 -- all_gather + cat along dim 0, rank-major."""
    return np.concatenate([np.ascontiguousarray(x) for x in xs], axis=0)


def get_local_id(ids: np.ndarray, rank: int, world: int) -> np.ndarray:
    """moco/util.py:95-97 -- ``ids.chunk(world)[rank]``."""
    n = ids.shape[0] // world
    return ids[rank * n:(rank + 1) * n]


def forward_shuffle(xs: Sequence[np.ndarray], epoch: int) -> Tuple[List[np.ndarray], np.ndarray]:
    """moco/util.py:69-79 for every rank at once.

    ``xs[r]`` is rank r's local batch.  Returns (per-rank shuffled batches,
    backward_inds).
    """
    world = len(xs)
    x_all = dist_collect(xs)
    fwd, bwd = get_shuffle_ids(x_all.shape[0], epoch)
    outs = [x_all[get_local_id(fwd, r, world)] for r in range(world)]
    return outs, bwd


def backward_shuffle(xs: Sequence[np.ndarray], backward_inds: np.ndarray,
                     return_local: bool = True):
    """moco/util.py:81-93 for every rank at once.

    Returns (x_all_unshuffled, [x_local per rank]) or x_all_unshuffled.
    """
    world = len(xs)
    x_all = dist_collect(xs)
    unshuf = x_all[backward_inds]
    if not return_local:
        return unshuf
    locals_ = [x_all[get_local_id(backward_inds, r, world)] for r in range(world)]
    return unshuf, locals_


# --------------------------------------------------------------------------
# MemoryMoCo + NCESoftmaxLoss  (reference moco/NCE/Contrast.py, NCECriterion.py)
# --------------------------------------------------------------------------


def queue_init_bound(feature_dim: int) -> float:
    """moco/NCE/Contrast.py:16 -- stdv = 1/sqrt(feature_dim/3)."""
    return 1.0 / math.sqrt(feature_dim / 3)


def enqueue_ids(index: int, all_size: int, queue_size: int) -> np.ndarray:
    """moco/NCE/Contrast.py:32 -- fmod(arange(all_size) + index, queue_size)."""
    return np.fmod(np.arange(all_size, dtype=np.int64) + index, queue_size)


class MemoryMoCoOracle:
    """moco/NCE/Contrast.py:6-36 in numpy (fp32 like the reference)."""

    def __init__(self, memory: np.ndarray, temperature: float = 0.07, index: int = 0):
        self.memory = np.array(memory, dtype=np.float32, copy=True)
        self.queue_size = self.memory.shape[0]
        self.temperature = temperature
        self.index = index

    def logits(self, q: np.ndarray, k: np.ndarray) -> np.ndarray:
        """Contrast.py:21-27 (no queue mutation)."""
        q = q.astype(np.float32)
        k = k.astype(np.float32)
        l_pos = (q * k).sum(axis=-1, keepdims=True)                  # :23
        l_neg = q @ self.memory.T                                     # :25 (pre-update snapshot)
        out = np.concatenate([l_pos, l_neg], axis=1)                  # :26
        return np.ascontiguousarray(out / np.float32(self.temperature))  # :27

    def enqueue(self, k_all: np.ndarray) -> np.ndarray:
        """Contrast.py:30-34; returns the ids written (for bit-exact checks)."""
        all_size = k_all.shape[0]
        ids = enqueue_ids(self.index, all_size, self.queue_size)
        # index_copy_ with duplicate ids (all_size > K) is order-dependent in
        # torch; the reference assumes all_size <= K (SURVEY S10).  numpy's
        # fancy assignment applies in order, matching the sequential semantics.
        for i, dst in enumerate(ids):
            self.memory[dst] = k_all[i]
        self.index = (self.index + all_size) % self.queue_size
        return ids

    def forward(self, q, k, k_all) -> np.ndarray:
        out = self.logits(q, k)
        self.enqueue(np.asarray(k_all, dtype=np.float32))
        return out


def logsumexp_rows(x: np.ndarray) -> np.ndarray:
    m = x.max(axis=1, keepdims=True)
    return (m + np.log(np.exp(x - m).sum(axis=1, keepdims=True)))[:, 0]


def nce_softmax_loss(out: np.ndarray) -> float:
    """moco/NCE/NCECriterion.py:11-13 -- CrossEntropyLoss(out, label 0), mean."""
    x = out.astype(np.float64)
    return float((logsumexp_rows(x) - x[:, 0]).mean())


def nce_rows(out: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Per-row (lse, loss, prob) -- loss_i = lse_i - x_i0; prob_i = exp(x_i0 - lse_i)."""
    x = out.astype(np.float64)
    lse = logsumexp_rows(x)
    return lse, lse - x[:, 0], np.exp(x[:, 0] - lse)


def prob_metric(out: np.ndarray) -> float:
    """train.py:264 -- softmax(out, 1)[:, 0].mean()."""
    return float(nce_rows(out)[2].mean())


def nce_backward_dq(q: np.ndarray, k: np.ndarray, memory_pre: np.ndarray,
                    temperature: float, grad_loss: float = 1.0) -> np.ndarray:
    """Autograd of train.py:262-263,273 w.r.t. q only (k, memory detached,
    Contrast.py:21,25):  dx_ij = (softmax_ij - [j==0]) / N,
    dq_i = (1/T) * (dx_i0 * k_i + sum_j dx_i,j+1 * memory_pre[j])."""
    q64, k64, m64 = (a.astype(np.float64) for a in (q, k, memory_pre))
    n = q.shape[0]
    x = np.concatenate([(q64 * k64).sum(-1, keepdims=True), q64 @ m64.T], axis=1) / temperature
    lse = logsumexp_rows(x)
    p = np.exp(x - lse[:, None])
    p[:, 0] -= 1.0
    dx = p * (grad_loss / n)
    dq = (dx[:, :1] * k64 + dx[:, 1:] @ m64) / temperature
    return dq


def nce_backward_dense(grad_out: np.ndarray, k: np.ndarray, memory_pre: np.ndarray,
                       temperature: float) -> np.ndarray:
    """Backward of Contrast.py:23-27 for an arbitrary upstream dense grad."""
    g = grad_out.astype(np.float64) / temperature
    return g[:, :1] * k.astype(np.float64) + g[:, 1:] @ memory_pre.astype(np.float64)


# --------------------------------------------------------------------------
# helpers shared by tests
# --------------------------------------------------------------------------


def bf16_round(x: np.ndarray) -> np.ndarray:
    """Round-to-nearest-even fp32 -> bf16 -> fp32 (so GPU and oracle see the
    same bf16-representable inputs; SURVEY §7 'bf16 parity definition')."""
    a = np.ascontiguousarray(x, dtype=np.float32)
    u = a.view(np.uint32).astype(np.uint64)
    rounded = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return (rounded & 0xFFFFFFFF).astype(np.uint32).view(np.float32).reshape(a.shape)


def l2_normalize(x: np.ndarray) -> np.ndarray:
    """moco/models/resnet.py:30-33 -- x / sqrt(sum x^2)."""
    return x / np.sqrt((x * x).sum(axis=1, keepdims=True))


# --------------------------------------------------------------------------
# Normalize layer in front of the head (SURVEY 8 f2).
# --------------------------------------------------------------------------
def normalize_backward(x: np.ndarray, grad_out: np.ndarray) -> np.ndarray:
    """Gradient through the reference's Normalize layer (moco/models/resnet.py:30-33, out = x / sqrt(sum x^2)):
    dx = (g - x^ <x^, g>) / |x| with x^ = x / |x| (what autograd produces for pow / sum / pow / div)."""
    x64, g64 = x.astype(np.float64), grad_out.astype(np.float64)
    nrm = np.sqrt((x64 * x64).sum(1, keepdims=True))
    xh = x64 / nrm
    return ((g64 - xh * (xh * g64).sum(1, keepdims=True)) / nrm)


def head_with_normalize(xq: np.ndarray, xk: np.ndarray, memory_pre: np.ndarray, T: float,
                        round_q_to_bf16: bool = False):
    """Normalize (resnet.py:24-33) -> MemoryMoCo logits (Contrast.py:20-27) -> NCESoftmaxLoss (NCECriterion.py:11-13)
    -> prob (train.py:264) -> gradient w.r.t. the RAW xq (train.py:273).  Returns (loss, prob, dxq, q^, k^).
    round_q_to_bf16 mirrors the kernels' operand contract (include/moco_b200.h): the negatives use bf16(q^), the
    positive logit the fp32 q^ and k^."""
    q, k = l2_normalize(xq), l2_normalize(xk)
    qn = bf16_round(q) if round_q_to_bf16 else q
    x0 = (q.astype(np.float64) * k.astype(np.float64)).sum(1) / T
    neg = qn.astype(np.float64) @ memory_pre.astype(np.float64).T / T
    out = np.concatenate([x0[:, None], neg], 1)
    lse = logsumexp_rows(out)
    p = np.exp(out - lse[:, None])
    loss = float((lse - x0).mean())
    prob = float(p[:, 0].mean())
    N = q.shape[0]
    dq = ((p[:, :1] - 1.0) * k.astype(np.float64) + p[:, 1:] @ memory_pre.astype(np.float64)) / (T * N)
    return loss, prob, normalize_backward(xq, dq), q, k


# --------------------------------------------------------------------------
# Momentum update of the key encoder.
# --------------------------------------------------------------------------
def moment_update(params: Sequence[np.ndarray], params_ema: Sequence[np.ndarray], m: float) -> List[np.ndarray]:
    """moco/util.py:124-127: ``p2.data.mul_(m).add_(1 - m, p1)`` per parameter pair.

    fp32 arithmetic as PyTorch evaluates it: ``m`` and ``1 - m`` (computed in double) are each rounded to
    fp32; ``t = rn(p2 * m)``; ``p2 = fma(1 - m, p1, t)`` (ATen's add-with-alpha is one fused multiply-add on
    its vectorised CPU path and in its CUDA functor).  The fma is emulated in float64: the product of two
    fp32 values is exact there and the sum rounds once more to 53 bits before the final fp32 rounding."""
    m32 = np.float32(m)
    a32 = np.float32(1 - m)
    out = []
    for p, pe in zip(params, params_ema):
        t = (pe.astype(np.float32) * m32).astype(np.float32)
        r = t.astype(np.float64) + np.float64(a32) * p.astype(np.float64)
        out.append(r.astype(np.float32))
    return out


# --------------------------------------------------------------------------
# One-sweep restatement of the head (checks the ALGORITHM of the CUDA one-pass kernel on the CPU).
# --------------------------------------------------------------------------
def one_sweep_head(q: np.ndarray, k: np.ndarray, memory_pre: np.ndarray, T: float, tile: int = 128,
                   slices: int = 4) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """lse, prob and dq of the reference head (Contrast.py:20-27, NCECriterion.py:11-13, train.py:264,273)
    computed the way a one-sweep kernel with a per-slice stabiliser does: the queue is cut into `slices` runs of
    `tile`-row tiles; every (slice, row) keeps the row maximum of its FIRST tile as a fixed stabiliser m and accumulates
    l = sum 2^(x - m) and O = sum 2^(x - m) queue_j in fp32 with no rescaling; slices are merged afterwards.
    Mathematically identical to logsumexp / softmax-weighted sum; in fp32 it overflows (inf) when a later logit
    exceeds the first tile's maximum by more than ~88 nats -- exactly the CUDA kernel's documented contract."""
    q32, k32, mem = q.astype(np.float32), k.astype(np.float32), memory_pre.astype(np.float32)
    N, C = q32.shape
    K = mem.shape[0]
    log2e = np.float32(1.4426950408889634)
    scale2 = np.float32(1.0 / T) * log2e
    ntiles = (K + tile - 1) // tile
    slices = max(1, min(slices, ntiles))
    x0 = (q32 * k32).sum(1, dtype=np.float32) * scale2                       # positive logit, log2 domain
    parts = []
    with np.errstate(over="ignore", invalid="ignore"):
        for s in range(slices):
            t0, t1 = s * ntiles // slices, (s + 1) * ntiles // slices
            rows = mem[t0 * tile:min(t1 * tile, K)]
            x = (q32 @ rows.T).astype(np.float32) * scale2                   # [N, rows of this slice]
            m = x[:, :min(tile, x.shape[1])].max(1)                          # first tile only
            p = np.exp2(x - m[:, None]).astype(np.float32)
            parts.append((m, p.sum(1, dtype=np.float32), (p @ rows).astype(np.float32)))
        M = np.maximum(x0, np.max([m for m, _, _ in parts], axis=0))
        l = np.exp2(x0 - M)
        for m, ls, _ in parts:
            l = l + ls * np.exp2(m - M)
        lse2 = M + np.log2(l)
        prob = np.exp2(x0 - lse2)
        O = np.zeros((N, C), np.float32)
        for m, _, o in parts:
            O += o * np.exp2(m - lse2)[:, None]
        dq = (np.float32(1.0 / T) / np.float32(N)) * (O + (prob - 1.0)[:, None] * k32)
    return (lse2 / log2e).astype(np.float32), prob.astype(np.float32), dq.astype(np.float32)
