"""Test helpers: oracle evaluation in K-chunks (memory-light at full BASELINE sizes), golden-vector loading, and the
kernels torch.profiler sees a call launch."""
import os

import numpy as np

from oracle import moco_oracle as O


def profiled(fns, reset=None):
    """[(result of fn(), names of the kernels it ran, its moco_launch_count() delta) for fn in fns], from one
    torch.profiler window in which each fn() is called in turn and must launch nothing but this library's kernels.
    Memcpy and memset activities are not kernels and are left out.  A sentinel kernel precedes every call and follows
    the last; a window in which the profiler lost any of them is not evidence of anything, so it is redone (after
    reset() restores the inputs, for calls that are not idempotent)."""
    import pytest
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    from moco_b200 import _lib
    for attempt in range(3):
        if attempt and reset is not None:
            reset()
        torch.cuda.synchronize()
        calls = []
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for fn in fns:
                torch.cuda._sleep(1000)
                torch.cuda.synchronize()
                before = _lib.launches
                out = fn()
                torch.cuda.synchronize()
                calls.append((out, _lib.launches - before))
            torch.cuda._sleep(1000)
            torch.cuda.synchronize()
        kernels = sorted((ev for ev in prof.events()
                          if ev.device_type == DeviceType.CUDA and not ev.name.startswith(("Memcpy", "Memset"))),
                         key=lambda ev: ev.time_range.start)
        marks = [i for i, ev in enumerate(kernels) if "spin_kernel" in ev.name]
        if len(marks) == len(fns) + 1:
            break
    else:
        pytest.fail("torch.profiler lost sentinel kernels three times")
    return [(out, [ev.name for ev in kernels[a + 1:b]], counted)
            for (out, counted), a, b in zip(calls, marks, marks[1:])]


def oracle_head_chunked(q, k, memory, T, chunk=16384, want_dq=True):
    """(lse[N], loss, prob, dq[N,C]) of the reference head, evaluated with the oracle's own
    functions on column chunks of the queue and merged with the log-sum-exp identity
    logsumexp(concat(a, b)) = logaddexp(logsumexp(a), logsumexp(b))."""
    N, C = q.shape
    K = memory.shape[0]
    q64, k64 = q.astype(np.float64), k.astype(np.float64)
    x0 = (q64 * k64).sum(-1) / T
    lse = x0.copy()
    for j0 in range(0, K, chunk):
        part = O.MemoryMoCoOracle(memory[j0:j0 + chunk], T).logits(q, k)[:, 1:]      # Contrast.py:25-27
        lse = np.logaddexp(lse, O.logsumexp_rows(part.astype(np.float64)))
    loss = float((lse - x0).mean())
    prob_rows = np.exp(x0 - lse)
    dq = None
    if want_dq:
        acc = (prob_rows - 1.0)[:, None] * k64
        for j0 in range(0, K, chunk):
            m = memory[j0:j0 + chunk].astype(np.float64)
            p = np.exp(q64 @ m.T / T - lse[:, None])
            acc += p @ m
        dq = acc / (T * N)
    return lse, loss, float(prob_rows.mean()), dq


def rand_unit(rng, n, c):
    x = rng.standard_normal((n, c)).astype(np.float32)
    return O.bf16_round(O.l2_normalize(x))


CONTRAST_GOLDEN = ("contrast.npz", "contrast_c1head.npz")      # one set of vectors, split to keep each file < 1 MB


def load_contrast_golden(golden_dir):
    """The reference's MemoryMoCo / NCESoftmaxLoss vectors (tests/golden/gen_golden.py:gen_contrast) as one mapping."""
    out = {}
    for name in CONTRAST_GOLDEN:
        with np.load(os.path.join(golden_dir, name)) as z:
            out.update({k: z[k] for k in z.files})
    return out
