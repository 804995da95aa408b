"""moco_launch_count() against the device: for every entry point that launches kernels, and every argument that
changes how many, the count's delta over one call equals the kernels torch.profiler saw run, and the number the header
documents.  Buffers are allocated before the profiled window, which holds nothing but C-ABI calls.

moco_shuffle_gather_sync and moco_signal_barrier wait for their peers, so they are not called here, and their counts
are not checked against the profiler."""
import ctypes

import numpy as np
import pytest
import torch

from tests import helpers

pytestmark = pytest.mark.gpu

M, C = 2048, 128                       # BatchNorm / conv1x1 rows and channels
NB, H, W = 2, 16, 16                   # max-pool inputs [NB, H, W, C]
K, INV_T = 8192, 1 / 0.07


def _lib():
    from moco_b200 import _lib
    return _lib


def _sms():
    n = ctypes.c_int()
    assert _lib().load().moco_device_info(ctypes.byref(n), None, None) == 0
    return n.value


def _bf16(*shape):
    return torch.randn(*shape, device="cuda").bfloat16()


def _f32(*shape):
    return torch.randn(*shape, device="cuda")


def _ptr(t):
    return t.data_ptr() if t is not None else None


class _Bn:
    """One BatchNorm's device tensors and its moco_bn_layer."""

    def __init__(self, c=C):
        ones = lambda: torch.ones(c, device="cuda")
        self.t = [ones(), torch.zeros(c, device="cuda"), torch.zeros(c, device="cuda"), ones(),
                  torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros(c, device="cuda"), ones(),
                  torch.zeros(c, device="cuda"), torch.zeros(c, device="cuda")]
        g, b, rm, rv, nbt, sm, si, dg, db = (t.data_ptr() for t in self.t)
        self.layer = _lib().BnLayer(g, b, rm, rv, nbt, 0.1, 1e-5, sm, si, dg, db)
        self.ref = ctypes.byref(self.layer)


def _workspace():
    lib = _lib().load()
    n = max(lib.moco_bn_workspace_bytes(), lib.moco_conv1x1_workspace_bytes())
    return torch.zeros(n, dtype=torch.uint8, device="cuda"), n


# ---------------------------------------------------------------------------------------------------------------
# training BatchNorm, conv1x1, eval and pooling: (expected launches, call)
# ---------------------------------------------------------------------------------------------------------------
def _bn_cases():
    lib, L = _lib().load(), _lib()
    bn, sc = _Bn(), _Bn()
    ws, nws = _workspace()
    x, r, y, dy, dy2, dx, dr, g = (_bf16(M, C) for _ in range(8))
    mask = torch.zeros(M, C // 8, dtype=torch.uint8, device="cuda")
    w, h = _bf16(C, C), _bf16(M, C)
    xp, yp = _bf16(NB, H, W, C), _bf16(NB, H // 2, W // 2, C)
    dyp, dy2p, dxp = _bf16(NB, H // 2, W // 2, C), _bf16(NB, H // 2, W // 2, C), _bf16(NB, H, W, C)
    taps = torch.zeros(NB, H // 2, W // 2, C, dtype=torch.uint8, device="cuda")
    s, t, s2, t2, feat = _f32(C), _f32(C), _f32(C), _f32(C), _f32(NB, C)
    b = bn.layer
    p = _ptr
    cases = {
        "bn_fwd_train": (2, lambda: lib.moco_bn_fwd_train(
            p(x), None, p(y), M, C, b.gamma, b.beta, b.running_mean, b.running_var, b.num_batches_tracked, 0.1, 1e-5,
            1, b.save_mean, b.save_invstd, p(ws), nws, None)),
        "bn_bwd": (2, lambda: lib.moco_bn_bwd(
            p(dy), p(x), p(y), M, C, b.gamma, b.beta, b.save_mean, b.save_invstd, 1, 0, p(dx), None, b.dgamma, b.dbeta,
            p(ws), nws, None)),
        "bn_bwd_apply_given": (1, lambda: lib.moco_bn_bwd_apply_given(p(g), p(x), None, M, C, bn.ref, None, p(dx),
                                                                       None, None)),
        "bn_relu_maxpool_fwd_train": (2, lambda: lib.moco_bn_relu_maxpool_fwd_train(
            p(xp), p(yp), p(taps), NB, H, W, C, bn.ref, p(ws), nws, None)),
        "conv1x1_bn_stats": (1, lambda: lib.moco_conv1x1_bn_stats(p(x), p(w), p(h), M, C, C, bn.ref, p(ws), nws, None)),
        "conv1x1_dgrad_bn_bwd": (1, lambda: lib.moco_conv1x1_dgrad_bn_bwd(
            p(dy), p(w), p(g), M, C, C, p(x), p(mask), p(dy2), None, bn.ref, None, p(ws), nws, None)),
        "bn_eval_act": (1, lambda: lib.moco_bn_eval_act(p(x), None, p(y), M, C, p(s), p(t), 1, None, None, None)),
        "bn_eval_act_shortcut": (1, lambda: lib.moco_bn_eval_act(p(x), p(r), p(y), M, C, p(s), p(t), 1, p(s2), p(t2),
                                                                  None)),
        "bn_relu_maxpool_eval": (1, lambda: lib.moco_bn_relu_maxpool_eval(p(xp), p(yp), NB, H, W, C, p(s), p(t), None)),
        "bn_eval_act_avgpool": (1, lambda: lib.moco_bn_eval_act_avgpool(
            p(x), None, p(feat), NB, M // NB, C, p(s), p(t), 1, None, None, None)),
        "bn_eval_act_avgpool_shortcut": (1, lambda: lib.moco_bn_eval_act_avgpool(
            p(x), p(r), p(feat), NB, M // NB, C, p(s), p(t), 1, p(s2), p(t2), None)),
        "maxpool_fwd": (1, lambda: lib.moco_maxpool3x3s2_fwd(p(xp), p(yp), p(taps), NB, H, W, C, None)),
        "maxpool_bwd": (1, lambda: lib.moco_maxpool3x3s2_bwd(p(dyp), p(taps), p(dxp), NB, H, W, C, None)),
        "maxpool_bwd2": (1, lambda: lib.moco_maxpool3x3s2_bwd2(p(dyp), p(dy2p), p(taps), p(dxp), NB, H, W, C, None)),
    }
    for short, shortcut in (("", None), ("_shortcut", sc)):
        scr = shortcut.ref if shortcut else None
        cases["bn_add_relu_fwd_train" + short] = (3 if shortcut else 2, lambda scr=scr: lib.moco_bn_add_relu_fwd_train(
            p(x), p(r), p(y), p(mask), M, C, bn.ref, scr, p(ws), nws, None))
        cases["bn_add_relu_bwd" + short] = (2, lambda scr=scr: lib.moco_bn_add_relu_bwd(
            p(dy), p(x), p(r), p(mask), M, C, bn.ref, scr, p(dx), p(dr), p(ws), nws, None))
        cases["bn_add_relu_bwd2" + short] = (2, lambda scr=scr: lib.moco_bn_add_relu_bwd2(
            p(dy), p(dy2), p(x), p(r), p(mask), M, C, bn.ref, scr, p(dx), p(dr), p(ws), nws, None))
        for given in range(4):
            n = 1 + (not given & L.BN_STATS_GIVEN) + (shortcut is not None and not given & L.BN_SC_STATS_GIVEN)
            cases[f"bn_fwd_train_given_{given}{short}"] = (n, lambda scr=scr, given=given: lib.moco_bn_fwd_train_given(
                p(x), p(r), p(y), p(mask), M, C, 1, bn.ref, scr, given, p(ws), nws, None))
            cases[f"conv1x1_bn_add_relu_fwd_{given}{short}"] = (n, lambda scr=scr, given=given:
                                                                 lib.moco_conv1x1_bn_add_relu_fwd(
                p(x), p(w), p(r), p(y), p(mask), M, C, C, bn.ref, scr, given, p(ws), nws, None))
    return cases


# ---------------------------------------------------------------------------------------------------------------
# the replicated and the sharded head
# ---------------------------------------------------------------------------------------------------------------
class _Head:
    def __init__(self, N, C, f32=False, logits=False, dq=True, K=K):
        self.N, self.C, self.K = N, C, K
        qk = torch.float32 if f32 else torch.bfloat16
        self.q = torch.nn.functional.normalize(_f32(N, C), dim=1).to(qk)
        self.k = torch.nn.functional.normalize(_f32(N, C), dim=1).to(qk)
        self.queue = torch.nn.functional.normalize(_f32(K, C), dim=1).bfloat16()
        self.rows = [_f32(N) for _ in range(3)] + [_f32(2)]
        self.logits = _f32(N, K + 1) if logits else None
        self.dq = _f32(N, C) if dq else None
        lib = _lib().load()
        self.nws = int(lib.moco_nce_workspace_bytes(N, C, K))
        self.ws = torch.zeros(self.nws + 256, dtype=torch.uint8, device="cuda")
        self.wsp = self.ws.data_ptr() + (-self.ws.data_ptr()) % 256

    def dtype(self):
        return _lib().dtype_code(self.q)

    def fwd(self, flags):
        return _lib().load().moco_nce_fwd(
            _ptr(self.q), _ptr(self.k), self.dtype(), _ptr(self.queue), self.N, self.C, self.K, INV_T, _ptr(self.logits),
            *map(_ptr, self.rows), _ptr(self.dq), self.wsp, self.nws, flags, None)

    def step(self, k_all, n_all):
        return _lib().load().moco_nce_step(
            _ptr(self.q), _ptr(self.k), self.dtype(), 0, _ptr(self.queue), None, self.N, self.C, self.K, INV_T,
            _ptr(k_all), _lib().dtype_code(k_all), n_all, 0, None, *map(_ptr, self.rows), _ptr(self.dq), self.wsp,
            self.nws, 0, None)


# (N, C, flags, want dq, want logits, fp32 q) -> launches; `SMS` stands for 128 rows per SM
HEAD_ROWS = {
    "one_sweep": ((256, 128, 0, True, False, True), 2),                   # sweep + tail
    "one_sweep_bf16_copy": ((256, 256, 0, True, False, True), 3),         # + the bf16 copy of q
    "two_pass": ((256, 128, 512, True, False, False), 5),                 # prep, stats, combine, dq, dq_reduce
    "no_gradient": ((256, 128, 0, False, False, False), 3),               # the statistics pass only
    "dense_logits": ((256, 128, 0, True, True, False), 5),
    "C_not_64k": ((256, 100, 0, True, False, False), 2),                  # prep + CUDA-core rows
    "force_simt": ((256, 128, 1, True, False, False), 2),
    "one_block_per_sm": (("SMS", 128, 0, True, False, False), 2),         # still the one sweep
    "more_blocks_than_sms": (("SMS+1", 128, 0, True, False, False), 2),   # the CUDA-core kernel
    "more_blocks_than_sms_C256_f32": (("SMS+1", 256, 0, True, False, True), 2),   # its prep is the bf16 copy
    "more_blocks_than_sms_two_pass": (("SMS+1", 128, 512, True, False, False), 2),
}


def _head_cases():
    lib = _lib().load()
    cases = {}
    for name, ((N, c, flags, dq, logits, f32), n) in HEAD_ROWS.items():
        if isinstance(N, str):
            N = 128 * _sms() + (1 if N.endswith("+1") else 0)
        h = _Head(N, c, f32=f32, logits=logits, dq=dq)
        cases["nce_fwd_" + name] = (n, lambda h=h, flags=flags: h.fwd(flags))
    # moco_nce_step: the tail kernel enqueues at C = 128; at C = 192 (24 vectors a row) a separate kernel does
    for c, fused in ((128, True), (192, False)):
        h = _Head(256, c)
        k_all = _bf16(256, c)
        cases[f"nce_step_C{c}_enqueue"] = (2 if fused else 3, lambda h=h, k_all=k_all: h.step(k_all, 256))
        cases[f"nce_step_C{c}_no_enqueue"] = (2, lambda h=h, k_all=k_all: h.step(k_all, 0))
    h = _Head(256, 128)
    grad = _f32(256, K + 1)
    cases["nce_bwd_dense"] = (1, lambda: lib.moco_nce_bwd_dense(_ptr(grad), _ptr(h.k), h.dtype(), _ptr(h.queue), 256,
                                                                 128, K, INV_T, _ptr(h.dq), None))
    # the sharded chain at world 1: stats (prep, sweep, combine), merge, dq (one pass: the reduction alone), both
    # finishes
    L = _lib()
    for mode, flags, n in (("one_pass", L.NCE_ONE_PASS, 7), ("two_pass", 0, 8)):
        h = _Head(256, 128)
        ms = torch.empty(256, 2, device="cuda")
        o = _f32(256, 128)
        lse, loss_rows, prob_rows, loss_prob = map(_ptr, h.rows)
        peers = (ctypes.c_void_p * 1)(o.data_ptr())

        def chain(h=h, flags=flags, ms=ms, o=o, lse=lse, loss_rows=loss_rows, prob_rows=prob_rows,
                  loss_prob=loss_prob, peers=peers):
            d = h.dtype()
            rcs = [lib.moco_nce_shard_stats(_ptr(h.q), _ptr(h.k), d, _ptr(h.queue), 256, 128, K, INV_T, _ptr(ms),
                                            h.wsp, h.nws, flags, None),
                   lib.moco_nce_shard_merge(_ptr(ms), 1, 256, 128, INV_T, lse, loss_rows, prob_rows, loss_prob, h.wsp,
                                            h.nws, None),
                   lib.moco_nce_shard_dq(_ptr(h.q), d, _ptr(h.queue), lse, 256, 128, K, INV_T, _ptr(o), h.wsp, h.nws,
                                         flags, None),
                   lib.moco_nce_shard_dq_finish(_ptr(o), _ptr(h.k), d, prob_rows, 256, 128, INV_T, _ptr(h.dq), None),
                   lib.moco_nce_shard_dq_finish_peers(peers, 1, 0, _ptr(h.k), d, prob_rows, 256, 128, INV_T,
                                                      _ptr(h.dq), None)]
            return next((rc for rc in rcs if rc != 0), 0)
        cases["nce_shard_chain_" + mode] = (n, chain)
    return cases


# ---------------------------------------------------------------------------------------------------------------
# queue, input path, EMA, augmentation, ShuffleBN gather
# ---------------------------------------------------------------------------------------------------------------
def _other_cases():
    lib, L = _lib().load(), _lib()
    p = _ptr
    queue, queue_f32, k_all = _bf16(K, C), _f32(K, C), _bf16(256, C)
    src32, dst16 = _f32(K * C), torch.empty(K * C, dtype=torch.bfloat16, device="cuda")
    ema_a, ema_b = _f32(100_000), _f32(100_000)
    chunk = lib.moco_ema_chunk_elems()
    segs = torch.tensor([[ema_a.data_ptr(), ema_b.data_ptr(), ema_a.numel()]], dtype=torch.int64, device="cuda")
    n_chunks = -(-ema_a.numel() // chunk)
    prefix = torch.tensor([0, n_chunks], dtype=torch.int32, device="cuda")
    N, Hc = 8, 32
    images = _f32(N, 6, Hc, Hc)
    rows = torch.randperm(N, device="cuda")
    nhwc = torch.empty(N, Hc * Hc, 3, dtype=torch.bfloat16, device="cuda")
    s2d = torch.empty(N, Hc // 2 + 3, Hc // 2 + 3, 16, dtype=torch.bfloat16, device="cuda")
    stride = 6 * Hc * Hc
    cases = {
        "queue_enqueue": (1, lambda: lib.moco_queue_enqueue(p(queue), p(queue_f32), p(k_all), L.MOCO_BF16, 256, C, K,
                                                            100, None)),
        "queue_enqueue_shard": (1, lambda: lib.moco_queue_enqueue_shard(
            p(queue), p(queue_f32), p(k_all), L.MOCO_BF16, 256, C, 2 * K, 100, 0, K, None)),
        "f32_to_bf16": (1, lambda: lib.moco_f32_to_bf16(p(src32), p(dst16), src32.numel(), None)),
        "ema_update": (1, lambda: lib.moco_ema_update(p(segs), p(prefix), 1, n_chunks, 0.999, 0.001, None)),
        "crop_to_nhwc_bf16": (1, lambda: lib.moco_crop_to_nhwc_bf16(p(images), L.MOCO_F32, stride, p(nhwc), N, 3,
                                                                    Hc * Hc, None)),
        "crop_gather_nhwc_bf16": (1, lambda: lib.moco_crop_gather_nhwc_bf16(p(images), L.MOCO_F32, stride, p(rows),
                                                                            p(nhwc), N, 3, Hc * Hc, None)),
        "crop_s2d_bf16": (1, lambda: lib.moco_crop_s2d_bf16(p(images), L.MOCO_F32, stride, p(rows), p(s2d), N, Hc, Hc,
                                                            None)),
    }
    # two crops of one 48 x 40 image, one with every flag
    pixels = torch.randint(0, 256, (48 * 40 * 3,), dtype=torch.uint8, device="cuda")
    rec = np.zeros((2, 14), np.int32)
    rec[:, 2:10] = [48, 40, 4, 3, 30, 28, 0, 0b11100100]
    rec[1, 8] = L.AUG_GRAY | L.AUG_FLIP | L.AUG_JITTER
    rec[:, 10:14] = np.array([1.2, 0.8, 1.1, 0.05], np.float32).view(np.int32)
    crops = torch.from_numpy(rec).cuda()
    norm = (ctypes.c_float * 6)(0.485, 0.456, 0.406, 0.229, 0.224, 0.225)
    aug_out, means = _f32(2, 3, 32, 32), _f32(2)
    cases["augment_crops"] = (2, lambda: lib.moco_augment_crops(p(pixels), pixels.numel(), p(crops), 2, 32, 32, norm,
                                                                p(aug_out), L.MOCO_F32, p(means), None))
    # moco_shuffle_gather at world 1: one warp a row below 16 KB, bulk copies up to 400 KB, 16-byte loads above
    # that or with MOCO_GATHER_LDG, and nothing at all for no rows
    n_rows = 16
    gather_rows = torch.randperm(n_rows, device="cuda")
    for name, row_bytes, flags, n in (("small", 512, L.GATHER_AUTO, 1), ("bulk", 32 * 1024, L.GATHER_AUTO, 1),
                                      ("ldg_flag", 32 * 1024, L.GATHER_LDG, 1),
                                      ("ldg_large_rows", 3 * 224 * 224 * 4, L.GATHER_AUTO, 1),
                                      ("no_rows", 512, L.GATHER_AUTO, 0)):
        src = torch.randint(0, 256, (n_rows * row_bytes,), dtype=torch.uint8, device="cuda")
        cases["shuffle_gather_" + name] = (n, lambda src=src, dst=torch.empty_like(src), row_bytes=row_bytes,
                                           flags=flags, rows=0 if name == "no_rows" else n_rows: lib.moco_shuffle_gather(
            (ctypes.c_void_p * 1)(src.data_ptr()), 1, n_rows, p(gather_rows), rows, row_bytes, p(dst), flags, None))
    return cases


@pytest.mark.parametrize("cases", [_bn_cases, _head_cases, _other_cases], ids=["bn", "head", "other"])
def test_launch_count_is_what_ran(cases):
    cases = cases()
    results = helpers.profiled([call for _, call in cases.values()])
    wrong = {name: dict(rc=rc, expect=expect, counted=counted, kernels=kernels)
             for (name, (expect, _)), (rc, kernels, counted) in zip(cases.items(), results)
             if rc != 0 or not counted == len(kernels) == expect}
    assert not wrong, wrong
