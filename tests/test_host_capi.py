"""Argument validation of the C ABI (include/moco_b200.h) for the entry points the other host tests leave out, and the
order in which each family reports two faults at once.  Every call here is refused before the entry point's first CUDA
call, so no GPU is needed and nothing is ever launched on the fake pointers."""
import ctypes

import pytest

from moco_b200 import _lib

FAKE = 0x10000                      # 256-byte aligned, never dereferenced: validation fails first
INVALID, UNSUPPORTED, WORKSPACE = -1, -2, -3
F32, BF16 = _lib.MOCO_F32, _lib.MOCO_BF16


def _p(n):
    """The n-th fake operand: 64 KiB apart, so no two alias and each is 256-byte aligned."""
    return FAKE + n * 0x10000


def _ptrs(*values):
    return (ctypes.c_void_p * len(values))(*values)


def _layer(**kw):
    f = dict(gamma=_p(20), beta=_p(21), save_mean=_p(22), save_invstd=_p(23), dgamma=_p(24), dbeta=_p(25),
             momentum=0.1, eps=1e-5)
    f.update(kw)
    return _lib.BnLayer(**f)


_NORM = (ctypes.c_float * 6)(0.485, 0.456, 0.406, 0.229, 0.224, 0.225)
_US = ctypes.c_float()
_OUT_PTR = ctypes.c_void_p()
_HANDLE = ctypes.create_string_buffer(64)
_STATUS = (ctypes.c_uint32 * 4)()


def _defaults(lib):
    """A call per entry point with every argument valid, in the header's order; each row below spoils one or two."""
    nce_ws = lib.moco_nce_workspace_bytes(8, 128, 1024)
    bn_ws = lib.moco_bn_workspace_bytes()
    cv_ws = lib.moco_conv1x1_workspace_bytes()
    return {
        "moco_nce_fwd": dict(q=_p(1), k=_p(2), dtype=F32, queue=_p(3), N=8, C=128, K=1024, inv_T=14.0, logits=None,
                             lse=_p(4), loss_rows=_p(5), prob_rows=_p(6), loss_prob=_p(7), dq=_p(8), ws=_p(9),
                             wsb=nce_ws, flags=0, stream=None),
        "moco_nce_step": dict(q=_p(1), k=_p(2), dtype=F32, normalize=0, queue=_p(3), queue_f32=None, N=8, C=128,
                              K=1024, inv_T=14.0, k_all=_p(10), k_all_dtype=F32, n_all=8, index=0, index_dev=None,
                              lse=_p(4), loss_rows=_p(5), prob_rows=_p(6), loss_prob=_p(7), dq=_p(8), ws=_p(9),
                              wsb=nce_ws, flags=0, stream=None),
        "moco_nce_bwd_dense": dict(grad_logits=_p(1), k=_p(2), k_dtype=F32, queue=_p(3), N=8, C=128, K=1024,
                                   inv_T=14.0, dq=_p(4), stream=None),
        "moco_prof_sweep_window": dict(ws=_p(1), n_ctas=132, us_out=ctypes.pointer(_US), stream=None),
        "moco_prof_set_events": dict(kernel=0, start=None, stop=None),
        "moco_queue_enqueue": dict(queue=_p(1), queue_f32=None, k_all=_p(2), k_dtype=BF16, n_all=4, C=64, K=16,
                                   index=3, stream=None),
        "moco_queue_enqueue_shard": dict(shard=_p(1), shard_f32=None, k_all=_p(2), k_dtype=BF16, n_all=4, C=64, K=16,
                                         index=3, row0=0, rows=8, stream=None),
        "moco_nce_shard_stats": dict(q_all=_p(1), k_all=_p(2), dtype=BF16, shard=_p(3), N=8, C=128, Ks=1024,
                                     inv_T=14.0, ms_out=_p(4), ws=_p(9), wsb=nce_ws, flags=0, stream=None),
        "moco_nce_shard_dq": dict(q_all=_p(1), dtype=BF16, shard=_p(3), lse_all=_p(4), N=8, C=128, Ks=1024,
                                  inv_T=14.0, o_partial=_p(5), ws=_p(9), wsb=nce_ws, flags=0, stream=None),
        "moco_f32_to_bf16": dict(src=_p(1), dst=_p(2), n=16, stream=None),
        "moco_ema_update": dict(segs=_p(1), prefix=_p(2), n_segs=1, n_chunks=1, m=0.999, one_minus_m=0.001,
                                stream=None),
        "moco_crop_s2d_bf16": dict(src=_p(1), dtype=F32, stride=3 * 32 * 32, src_rows=None, dst=_p(2), N=2, H=32,
                                   W=32, stream=None),
        "moco_augment_crops": dict(pixels=_p(1), pixels_bytes=1000, crops=_p(2), n_crops=2, out_h=224, out_w=224,
                                   norm=_NORM, dst=_p(3), dst_dtype=BF16, crop_means=_p(4), stream=None),
        "moco_maxpool3x3s2_fwd": dict(x=_p(1), y=_p(2), taps=_p(3), N=2, H=9, W=9, C=64, stream=None),
        "moco_maxpool3x3s2_bwd": dict(dy=_p(1), taps=_p(3), dx=_p(2), N=2, H=9, W=9, C=64, stream=None),
        "moco_maxpool3x3s2_bwd2": dict(dy=_p(1), dy2=_p(4), taps=_p(3), dx=_p(2), N=2, H=9, W=9, C=64, stream=None),
        "moco_bn_fwd_train": dict(x=_p(1), res=None, y=_p(2), M=1024, C=64, gamma=_p(20), beta=_p(21), rm=None,
                                  rv=None, nbt=None, momentum=0.1, eps=1e-5, relu=1, save_mean=_p(22),
                                  save_invstd=_p(23), ws=_p(9), wsb=bn_ws, stream=None),
        "moco_bn_add_relu_bwd2": dict(dy=_p(1), dy2=_p(2), x=_p(3), res=None, mask=_p(4), M=1024, C=64,
                                      bn=_layer(), sc=None, dx=_p(5), dres=None, ws=_p(9), wsb=bn_ws, stream=None),
        "moco_bn_relu_maxpool_fwd_train": dict(x=_p(1), y=_p(2), taps=_p(3), N=2, H=9, W=9, C=64, bn=_layer(),
                                               ws=_p(9), wsb=bn_ws, stream=None),
        "moco_conv1x1_bn_stats": dict(x=_p(1), w=_p(2), y=_p(3), M=1024, Cin=64, Cout=64, bn=_layer(), ws=_p(9),
                                      wsb=cv_ws, stream=None),
        "moco_conv1x1_bn_add_relu_fwd": dict(x=_p(1), w=_p(2), res=_p(3), y=_p(4), mask=None, M=1024, Cin=64,
                                             Cout=64, bn=_layer(), sc=None, given=0, ws=_p(9), wsb=max(cv_ws, bn_ws),
                                             stream=None),
        "moco_conv1x1_dgrad_bn_bwd": dict(dh=_p(1), w=_p(2), g=_p(3), M=1024, Cin=256, Cout=64, x=_p(4), mask=_p(5),
                                          dy2=_p(6), x2=None, bn=_layer(), sc=None, ws=_p(9), wsb=cv_ws, stream=None),
        "moco_crop_to_nhwc_bf16": dict(src=_p(1), dtype=F32, stride=1024, dst=_p(2), N=2, C=3, HW=64, stream=None),
        "moco_crop_gather_nhwc_bf16": dict(src=_p(1), dtype=F32, stride=1024, src_rows=_p(3), dst=_p(2), N=2, C=3,
                                           HW=64, stream=None),
        "moco_shuffle_gather": dict(peers=_ptrs(_p(1), _p(2)), world=2, rows_per_rank=4, src_rows=_p(3), n_rows=8,
                                    row_bytes=256, dst=_p(4), flags=0, stream=None),
        "moco_shuffle_gather_sync": dict(peers=_ptrs(_p(1), _p(2)), pads=_ptrs(_p(5), _p(6)), world=2, rank=0,
                                         epoch=1, rows_per_rank=4, src_rows=_p(3), n_rows=8, row_bytes=256,
                                         dst=_p(4), flags=0, stream=None),
        "moco_signal_barrier": dict(pads=_ptrs(_p(5), _p(6)), world=2, rank=0, epoch=1, stream=None),
        "moco_p2p_last_timeout": dict(out=_STATUS),
        "moco_p2p_alloc": dict(bytes=4096, out=ctypes.pointer(_OUT_PTR), handle=ctypes.addressof(_HANDLE)),
        "moco_p2p_open": dict(handle=ctypes.addressof(_HANDLE), out=ctypes.pointer(_OUT_PTR)),
    }


# (entry point, the spoiled arguments, expected return code, a substring of moco_last_error())
ROWS = [
    # ---- one fault
    *[("moco_nce_bwd_dense", kw, INVALID, b"moco_nce_bwd_dense: bad argument")
      for kw in (dict(grad_logits=None), dict(k=None), dict(queue=None), dict(dq=None), dict(N=0), dict(C=0),
                 dict(K=-1))],
    *[("moco_prof_sweep_window", kw, INVALID, b"moco_prof_sweep_window: bad argument")
      for kw in (dict(ws=None), dict(us_out=None), dict(n_ctas=0), dict(n_ctas=161))],
    *[("moco_prof_set_events", kw, INVALID, b"moco_prof_set_events: bad kernel id")
      for kw in (dict(kernel=-1), dict(kernel=3))],
    ("moco_queue_enqueue", dict(queue=None), INVALID, b"moco_queue_enqueue: bad argument"),
    ("moco_queue_enqueue", dict(index=16), INVALID, b"moco_queue_enqueue: bad argument"),
    ("moco_queue_enqueue", dict(n_all=17, index=3), INVALID, b"moco_queue_enqueue: n_all (17) > K (16)"),
    *[("moco_queue_enqueue_shard", kw, INVALID, b"moco_queue_enqueue_shard: bad argument")
      for kw in (dict(shard=None), dict(k_all=None), dict(row0=-1), dict(rows=0), dict(row0=9))],
    ("moco_queue_enqueue_shard", dict(n_all=17), INVALID, b"moco_queue_enqueue_shard: "),
    *[(entry, kw, INVALID, entry.encode() + b": bad argument")
      for entry in ("moco_nce_shard_stats", "moco_nce_shard_dq")
      for kw in (dict(q_all=None), dict(ws=None), dict(N=0), dict(C=0), dict(Ks=0), dict(ws=_p(9) + 16))],
    *[(entry, dict(wsb=kw), WORKSPACE, entry.encode() + b": workspace too small")
      for entry in ("moco_nce_shard_stats", "moco_nce_shard_dq") for kw in (0, 4096)],
    *[("moco_f32_to_bf16", kw, INVALID, b"moco_f32_to_bf16: null pointer") for kw in (dict(src=None), dict(dst=None))],
    *[("moco_ema_update", kw, INVALID, b"moco_ema_update: bad argument")
      for kw in (dict(n_segs=-1), dict(n_chunks=-1), dict(segs=None), dict(prefix=None))],
    *[("moco_crop_s2d_bf16", kw, INVALID, b"moco_crop_s2d_bf16: bad argument")
      for kw in (dict(N=-1), dict(dst=None), dict(src=None), dict(dtype=7), dict(stride=3 * 32 * 32 - 2),
                 dict(src=_p(1) + 4), dict(dst=_p(2) + 8), dict(stride=3 * 32 * 32 + 1))],
    *[("moco_crop_s2d_bf16", kw, UNSUPPORTED, b"moco_crop_s2d_bf16: needs even H, W >= 2")
      for kw in (dict(H=31), dict(W=1))],
    *[(entry, kw, INVALID, entry.encode() + b": bad argument")
      for entry in ("moco_crop_to_nhwc_bf16", "moco_crop_gather_nhwc_bf16")
      for kw in (dict(N=-1), dict(dst=None), dict(src=None), dict(dtype=7), dict(stride=3 * 64 - 4),
                 dict(src=_p(1) + 8), dict(dst=_p(2) + 8), dict(stride=1026), dict(dtype=BF16, stride=1028))],
    *[(entry, kw, UNSUPPORTED, entry.encode() + b": needs C <= 4 and H*W % 8 == 0")
      for entry in ("moco_crop_to_nhwc_bf16", "moco_crop_gather_nhwc_bf16") for kw in (dict(C=5), dict(HW=60))],
    *[("moco_maxpool3x3s2_fwd", kw, INVALID, b"moco_maxpool3x3s2_fwd: null or misaligned pointer")
      for kw in (dict(x=None), dict(y=_p(2) + 8), dict(taps=_p(3) + 4))],
    *[("moco_maxpool3x3s2_bwd", kw, INVALID, b"moco_maxpool3x3s2_bwd: null or misaligned pointer")
      for kw in (dict(dy=_p(1) + 8), dict(dx=None), dict(taps=_p(3) + 4))],
    *[("moco_maxpool3x3s2_bwd2", kw, INVALID, b"moco_maxpool3x3s2_bwd2: null or misaligned pointer")
      for kw in (dict(dy2=None), dict(dy2=_p(4) + 8), dict(dx=_p(2) + 8), dict(taps=None))],
    *[(entry, kw, UNSUPPORTED, entry.encode() + b": needs N, H, W >= 1 and C % 8 == 0")
      for entry in ("moco_maxpool3x3s2_fwd", "moco_maxpool3x3s2_bwd", "moco_maxpool3x3s2_bwd2")
      for kw in (dict(C=12), dict(N=0))],
    *[("moco_shuffle_gather", kw, INVALID, b"moco_shuffle_gather: bad argument")
      for kw in (dict(peers=None), dict(src_rows=None), dict(dst=None), dict(world=0), dict(world=17),
                 dict(rows_per_rank=0), dict(n_rows=-1), dict(row_bytes=0), dict(row_bytes=24), dict(dst=_p(4) + 8))],
    ("moco_shuffle_gather", dict(peers=_ptrs(_p(1), None)), INVALID, b"moco_shuffle_gather: peer 1"),
    ("moco_shuffle_gather", dict(peers=_ptrs(_p(1) + 8, _p(2))), INVALID, b"moco_shuffle_gather: peer 0"),
    *[("moco_shuffle_gather_sync", kw, INVALID, b"moco_shuffle_gather_sync: bad synchronisation argument")
      for kw in (dict(pads=None), dict(rank=-1), dict(rank=2), dict(epoch=0))],
    # the sync entry's own arguments are checked first; the gather's are the plain entry's checks
    *[("moco_shuffle_gather_sync", kw, INVALID, b"moco_shuffle_gather")
      for kw in (dict(rows_per_rank=0), dict(row_bytes=24), dict(peers=_ptrs(None, _p(2))))],
    *[("moco_signal_barrier", kw, INVALID, b"moco_signal_barrier: bad argument")
      for kw in (dict(pads=None), dict(world=0), dict(world=17), dict(rank=-1), dict(rank=2))],
    ("moco_p2p_last_timeout", dict(out=None), INVALID, b"moco_p2p_last_timeout"),
    *[("moco_p2p_alloc", kw, INVALID, b"moco_p2p_alloc: bad argument")
      for kw in (dict(bytes=0), dict(out=None), dict(handle=None))],
    *[("moco_p2p_open", kw, INVALID, b"moco_p2p_open: bad argument") for kw in (dict(handle=None), dict(out=None))],

    # ---- two faults: which one each family reports
    # BatchNorm training: the arguments, then the workspace, then the launcher's shape envelope
    ("moco_bn_fwd_train", dict(x=None, wsb=0), INVALID, b"moco_bn_fwd_train: bad argument"),
    ("moco_bn_fwd_train", dict(wsb=0, C=96), WORKSPACE, b"moco_bn_fwd_train: workspace too small"),
    ("moco_bn_fwd_train", dict(C=96), UNSUPPORTED, b"moco_bn_fwd_train: needs M >= 1 and C a power of two"),
    ("moco_bn_add_relu_bwd2", dict(dy2=None, wsb=0), INVALID, b"moco_bn_add_relu_bwd2: bad argument"),
    ("moco_bn_add_relu_bwd2", dict(wsb=0, M=0), WORKSPACE, b"moco_bn_add_relu_bwd2: workspace too small"),
    ("moco_bn_relu_maxpool_fwd_train", dict(taps=None, wsb=0), INVALID, b"moco_bn_relu_maxpool_fwd_train: bad argument"),
    ("moco_bn_relu_maxpool_fwd_train", dict(wsb=0, C=72), WORKSPACE, b"moco_bn_relu_maxpool_fwd_train: workspace"),
    ("moco_bn_relu_maxpool_fwd_train", dict(H=0), UNSUPPORTED, b"moco_bn_relu_maxpool_fwd_train: needs N, H, W >= 1"),
    # conv1x1: the arguments, then the shape envelope, then the workspace
    *[(entry, dict(kw, M=0), INVALID, entry.encode() + b": bad argument")
      for entry, kw in (("moco_conv1x1_bn_stats", dict(x=None)), ("moco_conv1x1_bn_add_relu_fwd", dict(y=_p(1))),
                        ("moco_conv1x1_dgrad_bn_bwd", dict(g=_p(1))))],
    *[(entry, dict(M=0, wsb=0), UNSUPPORTED, entry.encode() + b": needs ")
      for entry in ("moco_conv1x1_bn_stats", "moco_conv1x1_bn_add_relu_fwd", "moco_conv1x1_dgrad_bn_bwd")],
    ("moco_conv1x1_bn_stats", dict(Cout=96), UNSUPPORTED, b"Cout a multiple of 64 in [64, 4096]"),
    ("moco_conv1x1_bn_add_relu_fwd", dict(Cout=192), UNSUPPORTED, b"Cout a power of two in [64, 2048]"),
    ("moco_conv1x1_dgrad_bn_bwd", dict(Cin=64), UNSUPPORTED, b"Cin a power of two in [128, 2048]"),
    *[(entry, dict(wsb=0), WORKSPACE, entry.encode() + b": workspace too small")
      for entry in ("moco_conv1x1_bn_stats", "moco_conv1x1_bn_add_relu_fwd", "moco_conv1x1_dgrad_bn_bwd")],
    # NCE head: null / size, then the workspace's 256-byte alignment, then the operands' 16-byte alignment, then the
    # workspace size; moco_nce_step checks its enqueue arguments before all of these
    ("moco_nce_fwd", dict(q=None, ws=_p(9) + 16), INVALID, b"moco_nce_fwd: null pointer"),
    ("moco_nce_fwd", dict(N=0, ws=_p(9) + 16), INVALID, b"moco_nce_fwd: bad N/C/K/inv_T/dtype"),
    ("moco_nce_fwd", dict(ws=_p(9) + 16, q=_p(1) + 8), INVALID, b"moco_nce_fwd: workspace must be 256-byte aligned"),
    ("moco_nce_fwd", dict(q=_p(1) + 8, wsb=0), INVALID, b"moco_nce_fwd: q, the queue and k_all must be 16-byte"),
    ("moco_nce_fwd", dict(wsb=4096), WORKSPACE, b"moco_nce_fwd: workspace too small"),
    ("moco_nce_step", dict(n_all=1025, q=None), INVALID, b"moco_nce_step: bad enqueue argument"),
    ("moco_nce_step", dict(k_all=_p(10) + 8, ws=_p(9) + 16), INVALID, b"moco_nce_step: workspace must be 256-byte"),
    ("moco_nce_step", dict(k_all=_p(10) + 8, wsb=0), INVALID, b"moco_nce_step: q, the queue and k_all must be 16-byte"),
    # the sharded head: shard_common's checks and workspace size come before the entry's own null-pointer check
    *[(entry, dict(kw, wsb=0), WORKSPACE, entry.encode() + b": workspace too small")
      for entry, kws in (("moco_nce_shard_stats", (dict(k_all=None), dict(shard=None), dict(ms_out=None))),
                         ("moco_nce_shard_dq", (dict(shard=None), dict(lse_all=None), dict(o_partial=None))))
      for kw in kws],
    ("moco_nce_shard_stats", dict(q_all=None, wsb=0), INVALID, b"moco_nce_shard_stats: bad argument"),
    # augment: a shape outside the envelope is a bad argument, reported after the pointers and dtype
    ("moco_augment_crops", dict(out_h=0), INVALID, b"moco_augment_crops: needs n_crops in [0, 65535]"),
    ("moco_augment_crops", dict(n_crops=-1), INVALID, b"moco_augment_crops: needs n_crops in [0, 65535]"),
    ("moco_augment_crops", dict(dst_dtype=7, out_h=0), INVALID, b"moco_augment_crops: bad argument"),
]


def _call(lib, defaults, entry, kw):
    args = dict(defaults[entry])
    assert set(kw) <= set(args), (entry, kw)
    args.update(kw)
    return getattr(lib, entry)(*args.values())


def test_every_row_spoils_a_known_argument_and_the_defaults_cover_the_header():
    lib = _lib.load()
    defaults = _defaults(lib)
    for entry, args in defaults.items():
        assert len(args) == len(_lib.SIGNATURES[entry][1]), entry
    assert {r[0] for r in ROWS} == set(defaults)


@pytest.mark.parametrize("entry", sorted({r[0] for r in ROWS}))
def test_refusals_before_any_cuda_call(entry):
    lib = _lib.load()
    defaults = _defaults(lib)
    before = _lib.launches
    for e, kw, rc, msg in ROWS:
        if e != entry:
            continue
        got = _call(lib, defaults, e, kw)
        err = lib.moco_last_error()
        assert (got, msg in err) == (rc, True), (e, kw, got, err)
    assert _lib.launches == before
