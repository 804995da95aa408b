"""ctypes binding of libmoco_b200.so (the C ABI in include/moco_b200.h).

The library is built in-tree by ``moco_b200/build.py`` (nvcc, sm_90a).  There is
no CPU fallback: if the shared object is missing and cannot be built, importing
any compute entry point raises.

``load()`` returns the ``ctypes.CDLL`` itself.  ``launches`` reads ``moco_launch_count()``: the kernels the library
has launched in this process, counted in C where each kernel is launched.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_int64, c_size_t, c_uint32, c_ulonglong, c_void_p

from . import build as _build

ABI_VERSION = 3                    # MOCO_B200_ABI_VERSION (include/moco_b200.h)
MOCO_F32, MOCO_BF16 = 0, 1
NCE_AUTO, NCE_FORCE_SIMT, NCE_CTA_PAIR, NCE_SINGLE_CTA = 0, 1, 2, 4
NCE_TWO_PASS, NCE_ONE_PASS = 512, 1024
ONE_PASS_MAX_INV_T = 25.0          # MOCO_ONE_PASS_MAX_INV_T (include/moco_b200.h)
GATHER_AUTO, GATHER_LDG = 0, 1
BN_STATS_GIVEN, BN_SC_STATS_GIVEN = 1, 2    # moco_bn_fwd_train_given `stats_given` bits
AUG_GRAY, AUG_FLIP, AUG_JITTER = 1, 2, 4    # moco_aug_crop `flags` bits
ERR_CAPACITY = -5                  # MOCO_ERR_CAPACITY: moco_knn needs a larger workspace



class BnLayer(ctypes.Structure):
    """moco_bn_layer (include/moco_b200.h): one BatchNorm's device pointers and hyper-parameters."""
    _fields_ = [("gamma", c_void_p), ("beta", c_void_p), ("running_mean", c_void_p), ("running_var", c_void_p),
                ("num_batches_tracked", c_void_p), ("momentum", c_float), ("eps", c_float),
                ("save_mean", c_void_p), ("save_invstd", c_void_p), ("dgamma", c_void_p), ("dbeta", c_void_p)]


# every symbol include/moco_b200.h declares: name -> (restype, argtypes)
SIGNATURES = {
    "moco_abi_version": (c_int, []),
    "moco_last_error": (c_char_p, []),
    "moco_device_info": (c_int, [POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    "moco_launch_count": (c_ulonglong, []),
    "moco_nce_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "moco_nce_fwd": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_float,
                             c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                             c_void_p, c_size_t, c_int, c_void_p]),
    "moco_nce_step": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_float,
                              c_void_p, c_int, c_int, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                              c_void_p, c_size_t, c_int, c_void_p]),
    "moco_prof_sweep_window": (c_int, [c_void_p, c_int, POINTER(c_float), c_void_p]),
    "moco_prof_set_events": (c_int, [c_int, c_void_p, c_void_p]),
    "moco_nce_bwd_dense": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_float,
                                   c_void_p, c_void_p]),
    "moco_queue_enqueue": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int64, c_int64, c_void_p]),
    "moco_nce_shard_stats": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_float, c_void_p,
                                     c_void_p, c_size_t, c_int, c_void_p]),
    "moco_nce_shard_merge": (c_int, [c_void_p, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_size_t, c_void_p]),
    "moco_nce_shard_dq": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_void_p,
                                  c_void_p, c_size_t, c_int, c_void_p]),
    "moco_nce_shard_dq_finish": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_float, c_void_p, c_void_p]),
    "moco_nce_shard_dq_finish_peers": (c_int, [POINTER(c_void_p), c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_int,
                                               c_float, c_void_p, c_void_p]),
    "moco_queue_enqueue_shard": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int64, c_int64,
                                         c_int64, c_int64, c_void_p]),
    "moco_f32_to_bf16": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "moco_ema_chunk_elems": (c_int, []),
    "moco_ema_update": (c_int, [c_void_p, c_void_p, c_int, c_int, c_float, c_float, c_void_p]),
    "moco_crop_s2d_bf16": (c_int, [c_void_p, c_int, c_int64, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "moco_maxpool3x3s2_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "moco_maxpool3x3s2_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "moco_maxpool3x3s2_bwd2": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "moco_bn_workspace_bytes": (c_size_t, []),
    "moco_bn_fwd_train": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_void_p, c_float, c_float, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "moco_bn_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                            c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "moco_bn_add_relu_fwd_train": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, POINTER(BnLayer),
                                           POINTER(BnLayer), c_void_p, c_size_t, c_void_p]),
    "moco_bn_add_relu_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, POINTER(BnLayer),
                                     POINTER(BnLayer), c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "moco_bn_add_relu_bwd2": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int,
                                      POINTER(BnLayer), POINTER(BnLayer), c_void_p, c_void_p, c_void_p, c_size_t,
                                      c_void_p]),
    "moco_bn_fwd_train_given": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, POINTER(BnLayer),
                                        POINTER(BnLayer), c_int, c_void_p, c_size_t, c_void_p]),
    "moco_conv1x1_workspace_bytes": (c_size_t, []),
    "moco_conv1x1_bn_stats": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, POINTER(BnLayer), c_void_p,
                                      c_size_t, c_void_p]),
    "moco_conv1x1_bn_add_relu_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int,
                                             POINTER(BnLayer), POINTER(BnLayer), c_int, c_void_p, c_size_t,
                                             c_void_p]),
    "moco_conv1x1_dgrad_bn_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p,
                                          c_void_p, c_void_p, POINTER(BnLayer), POINTER(BnLayer), c_void_p, c_size_t,
                                          c_void_p]),
    "moco_bn_bwd_apply_given": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, POINTER(BnLayer),
                                        POINTER(BnLayer), c_void_p, c_void_p, c_void_p]),
    "moco_bn_relu_maxpool_fwd_train": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                               POINTER(BnLayer), c_void_p, c_size_t, c_void_p]),
    "moco_bn_eval_act": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_int, c_void_p,
                                 c_void_p, c_void_p]),
    "moco_bn_relu_maxpool_eval": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "moco_bn_eval_act_avgpool": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int,
                                         c_void_p, c_void_p, c_void_p]),
    "moco_knn_workspace_bytes": (c_size_t, [c_int, c_int64, c_int64]),
    "moco_knn": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int64, c_int, c_int, c_float, c_int, c_void_p, c_void_p,
                         c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, POINTER(c_int64), c_void_p]),
    "moco_augment_crops": (c_int, [c_void_p, c_size_t, c_void_p, c_int, c_int, c_int, POINTER(c_float), c_void_p, c_int,
                                   c_void_p, c_void_p]),
    "moco_resize_center_crops": (c_int, [c_void_p, c_size_t, c_void_p, c_int, c_int, c_int, POINTER(c_float), c_void_p,
                                         c_int, c_void_p]),
    "moco_crop_to_nhwc_bf16": (c_int, [c_void_p, c_int, c_int64, c_void_p, c_int, c_int, c_int, c_void_p]),
    "moco_shuffle_gather": (c_int, [POINTER(c_void_p), c_int, c_int, c_void_p, c_int, c_size_t, c_void_p, c_int, c_void_p]),
    "moco_shuffle_gather_sync": (c_int, [POINTER(c_void_p), POINTER(c_void_p), c_int, c_int, c_uint32, c_int, c_void_p, c_int,
                                         c_size_t, c_void_p, c_int, c_void_p]),
    "moco_p2p_last_timeout": (c_int, [POINTER(c_uint32)]),
    "moco_crop_gather_nhwc_bf16": (c_int, [c_void_p, c_int, c_int64, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "moco_signal_barrier": (c_int, [POINTER(c_void_p), c_int, c_int, c_uint32, c_void_p]),
    "moco_p2p_alloc": (c_int, [c_size_t, POINTER(c_void_p), c_void_p]),
    "moco_p2p_open": (c_int, [c_void_p, POINTER(c_void_p)]),
    "moco_p2p_close": (c_int, [c_void_p]),
    "moco_p2p_free": (c_int, [c_void_p]),
}

_lib = None


def lib_path() -> str:
    return _build.LIB


def load() -> ctypes.CDLL:
    """Load (building first if needed and possible) libmoco_b200.so."""
    global _lib
    if _lib is not None:
        return _lib
    import torch  # noqa: F401  (loads the CUDA runtime the library links against)
    path = _build.LIB
    if not os.path.exists(path):
        try:
            _build.build()
        except Exception as exc:  # no nvcc on this box and no prebuilt library
            raise RuntimeError(
                f"moco_b200: {path} is missing and could not be built ({exc}); "
                "there is no CPU fallback for the CUDA hot path") from exc
    lib = ctypes.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    if lib.moco_abi_version() != ABI_VERSION:
        raise RuntimeError("moco_b200: ABI version mismatch between _lib.py and libmoco_b200.so")
    _lib = lib
    return _lib


def __getattr__(name):
    if name == "launches":             # bench.py reports the delta over its timed steps as `gpu_launches`
        return load().moco_launch_count()
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")


def check(code: int, what: str) -> None:
    if code != 0:
        msg = load().moco_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"moco_b200.{what} failed ({code}): {msg}")


def dtype_code(t) -> int:
    import torch
    if t.dtype == torch.float32:
        return MOCO_F32
    if t.dtype == torch.bfloat16:
        return MOCO_BF16
    raise TypeError(f"moco_b200: unsupported dtype {t.dtype} (expected float32 or bfloat16)")


def cur_stream() -> int:
    """torch.cuda.current_stream().cuda_stream of the current device, read without building a Stream object: it is
    called for every launch, and the Stream path's device-index helpers cost more host time than most launches."""
    import torch
    return torch._C._cuda_getCurrentRawStream(torch._C._cuda_getDevice())


def require_cuda(*tensors) -> None:
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("moco_b200: the contrastive hot path runs on CUDA only "
                               "(got a CPU tensor); there is no CPU fallback")
