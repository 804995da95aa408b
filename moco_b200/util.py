"""ShuffleBN and helpers -- drop-in for the hot-path part of ``moco/util.py`` (bl0/moco).

Same public names and semantics as the reference (``util.py:47-111``):
``dist_collect``, ``DistributedShufle.{forward_shuffle, backward_shuffle,
get_local_id, get_shuffle_ids}``; plus ``set_bn_train`` / ``moment_update``
(``util.py:114-127``) which the training step needs.

Native design: the reference all_gathers every rank's whole batch (W x the
bytes it needs, plus a zero-fill and a cat of the same size, util.py:55-58) and
then indexes it.  Here each rank publishes its batch in a peer-mapped staging
buffer and every rank PULLS exactly the rows its slice of the permutation names,
straight over NVLink/NVSwitch, with ONE kernel (``moco_shuffle_gather_sync``): the
permutation is the address computation, and the cross-GPU "everybody has published"
event is signalled and awaited inside that same kernel (peer-mapped signal pads,
time-bounded wait).  Staging buffers are double-buffered so one event per shuffle
suffices.  On a single GPU the forward permute of the images is folded into the
crop / cast / layout kernel (``moco_crop_gather_nhwc_bf16``).
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional, Tuple

import torch
import torch.distributed as dist

from . import _lib


def _world() -> Tuple[int, int]:
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


# ---------------------------------------------------------------------------
# permutation ids (host side; bit-exact with the reference)
# ---------------------------------------------------------------------------
_IDS_CACHE: Dict[Tuple[int, int, str], Tuple[torch.Tensor, torch.Tensor]] = {}


def shuffle_ids_cpu(bsz: int, epoch: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """forward/backward permutation exactly as ``util.py:99-111`` computes them
    (``torch.manual_seed(epoch); torch.randperm(bsz)`` on the CPU generator), but
    drawn from a PRIVATE generator: the reference re-seeds the global RNG on every
    training step as a side effect (SURVEY §5); we do not."""
    g = torch.Generator(device="cpu")
    g.manual_seed(epoch)
    forward_inds = torch.randperm(bsz, generator=g).long()
    backward_inds = torch.zeros(bsz, dtype=torch.long)
    backward_inds.index_copy_(0, forward_inds, torch.arange(bsz, dtype=torch.long))
    return forward_inds, backward_inds


def plan_forward(forward_inds: torch.Tensor, rank: int, world: int) -> torch.Tensor:
    """Global source rows rank `rank` pulls in forward_shuffle (util.py:77-79,96-97)."""
    n = forward_inds.shape[0] // world
    return forward_inds[rank * n:(rank + 1) * n]


# ---------------------------------------------------------------------------
# peer-memory context
# ---------------------------------------------------------------------------
class _PeerBuffer:
    """A cudaMalloc'ed buffer of this rank, mapped by every peer (CUDA IPC)."""

    def __init__(self, nbytes: int, rank: int, world: int, group=None):
        lib = _lib.load()
        self.nbytes = nbytes
        self.rank, self.world = rank, world
        ptr = ctypes.c_void_p()
        handle = (ctypes.c_ubyte * 64)()
        _lib.check(lib.moco_p2p_alloc(nbytes, ctypes.byref(ptr), handle), "moco_p2p_alloc")
        self.local = ptr.value
        self.ptrs = [None] * world
        self.ptrs[rank] = self.local
        if world > 1:
            handles = [None] * world
            dist.all_gather_object(handles, bytes(handle), group=group)
            for r in range(world):
                if r == rank:
                    continue
                h = (ctypes.c_ubyte * 64).from_buffer_copy(handles[r])
                p = ctypes.c_void_p()
                _lib.check(lib.moco_p2p_open(h, ctypes.byref(p)), "moco_p2p_open")
                self.ptrs[r] = p.value
        self.table = (ctypes.c_void_p * world)(*self.ptrs)
        self._views = {}

    def release(self):
        """Unmap the peers' buffers and free this rank's (collective in effect: every rank releases the same buffer at
        the same point; the caller orders it after the last use with a barrier)."""
        lib = _lib.load()
        for r, p in enumerate(self.ptrs):
            if p is not None and r != self.rank:
                lib.moco_p2p_close(p)
        if self.local is not None:
            lib.moco_p2p_free(self.local)
        self.ptrs, self.local = [None] * self.world, None
        self._views = {}

    def tensor(self, shape, dtype) -> torch.Tensor:
        """View of the local buffer as a torch tensor (no copy; cached per shape / dtype -- building one through
        __cuda_array_interface__ costs tens of microseconds of host time)."""
        key = (tuple(shape), dtype)
        hit = self._views.get(key)
        if hit is not None:
            return hit
        numel = 1
        for s in shape:
            numel *= s
        nbytes = numel * torch.empty((), dtype=dtype).element_size()
        assert nbytes <= self.nbytes

        class _Iface:
            pass
        obj = _Iface()
        obj.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1",
                                        "data": (self.local, False), "version": 2}
        t = torch.as_tensor(obj, device=f"cuda:{torch.cuda.current_device()}")
        out = self._views[key] = t.view(dtype).view(tuple(shape))
        return out


class ShuffleContext:
    """Per-process-group state of the P2P ShuffleBN: staging buffers (double-buffered), signal pad,
    barrier epoch.  Created lazily on first use; every rank must call the shuffles in the same order."""

    _instance: Optional["ShuffleContext"] = None

    def __init__(self, group=None):
        self.rank, self.world = _world()
        self.group = group
        self.pad = _PeerBuffer(4096, self.rank, self.world, group) if self.world > 1 else None
        self.epoch = 0
        self.staging: Dict[str, list] = {}
        self.turn: Dict[str, int] = {}
        self.gather_flags = _lib.GATHER_AUTO
        self._local_stage: Dict[str, torch.Tensor] = {}

    @classmethod
    def get(cls) -> "ShuffleContext":
        rank, world = _world()
        inst = cls._instance
        if inst is None or inst.world != world or inst.rank != rank:
            inst = cls._instance = ShuffleContext()
        return inst

    def _staging(self, kind: str, nbytes: int):
        bufs = self.staging.get(kind)
        if bufs is None or bufs[0].nbytes < nbytes:
            # (re)allocation is collective: every rank sees the same sizes at the same call
            if bufs is not None:
                # nobody may still be pulling from the old buffers: device-side event + host sync, then unmap / free
                self.barrier()
                torch.cuda.current_stream().synchronize()
                if self.world > 1:
                    dist.barrier(group=self.group)
                for b in bufs:
                    b.release()
            bufs = [_PeerBuffer(nbytes, self.rank, self.world, self.group) for _ in range(2)]
            self.staging[kind] = bufs
            self.turn[kind] = 0
        t = self.turn[kind]
        self.turn[kind] = t ^ 1
        return bufs[t]

    def barrier(self):
        lib = _lib.load()
        self.epoch += 1
        _lib.check(lib.moco_signal_barrier(self.pad.table, self.world, self.rank, self.epoch, _lib.cur_stream()),
                   "moco_signal_barrier")

    def _pull(self, table, n, src_rows, row_bytes, out_ptr, synced: bool):
        """The P2P pull.  synced=True: the "every peer has published" event rides in the SAME kernel
        (moco_shuffle_gather_sync) -- no separate barrier launch."""
        lib = _lib.load()
        if synced and self.world > 1:
            self.epoch += 1
            _lib.check(lib.moco_shuffle_gather_sync(table, self.pad.table, self.world, self.rank, self.epoch, n,
                                                    src_rows.data_ptr(), src_rows.shape[0], row_bytes, out_ptr,
                                                    self.gather_flags, _lib.cur_stream()), "moco_shuffle_gather_sync")
        else:
            _lib.check(lib.moco_shuffle_gather(table, self.world, n, src_rows.data_ptr(), src_rows.shape[0], row_bytes,
                                               out_ptr, self.gather_flags, _lib.cur_stream()), "moco_shuffle_gather")

    @staticmethod
    def last_timeout():
        """(timed_out, peer, event, waited_ms) of the last peer wait that expired in this process, or None."""
        lib = _lib.load()
        out = (ctypes.c_uint32 * 4)()
        if lib.moco_p2p_last_timeout(out) != 0 or out[0] == 0:
            return None
        return {"peer": int(out[1]), "event": int(out[2]), "waited_ms": int(out[3])}

    def gather(self, kind: str, x: torch.Tensor, src_rows: torch.Tensor, cast_dtype=None,
               channels_last: bool = False) -> torch.Tensor:
        """out[i] = (rank-major concatenation of every rank's x)[src_rows[i]].

        cast_dtype (world > 1 only): publish the batch in this dtype -- the cast is fused into the copy
        into the peer-visible staging buffer, so e.g. fp32 images cross NVLink as bf16 (what the autocast
        key encoder would round them to anyway).

        channels_last (images, SURVEY.md 8 f3): publish the batch as bf16 NHWC with ONE kernel
        (``moco_crop_to_nhwc_bf16``: crop selection from a wider NCHW batch, cast and layout change together) and
        return a bf16 ``channels_last`` tensor, so the first convolution of a channels_last encoder reads exactly
        the bytes that were gathered -- no ``.contiguous()``, cast or layout pass in between."""
        lib = _lib.load()
        _lib.require_cuda(x, src_rows)
        if channels_last:
            return self._gather_nhwc(kind, x, src_rows, s2d=(channels_last == "s2d"))
        x = x.contiguous()
        n = x.shape[0]
        dtype = cast_dtype if (cast_dtype is not None and self.world > 1) else x.dtype
        esize = torch.empty((), dtype=dtype).element_size()
        row_bytes = x[0].numel() * esize if n else 0
        if row_bytes % 16 != 0:
            raise ValueError(f"moco_b200 shuffle: row size {row_bytes} B is not a multiple of 16")
        out = torch.empty((src_rows.shape[0],) + tuple(x.shape[1:]), dtype=dtype, device=x.device)
        if self.world == 1:
            table = (ctypes.c_void_p * 1)(x.data_ptr())
        else:
            buf = self._staging(kind, x.numel() * esize)
            stage = buf.tensor(x.shape, dtype)
            if stage.data_ptr() != x.data_ptr():
                stage.copy_(x)
            table = buf.table        # "every rank's staging buffer is complete" rides in the pull kernel itself
        self._pull(table, n, src_rows, row_bytes, out.data_ptr(), synced=True)
        return out

    def _gather_nhwc(self, kind: str, x: torch.Tensor, src_rows: torch.Tensor, s2d: bool = False) -> torch.Tensor:
        lib = _lib.load()
        if x.dim() != 4:
            raise ValueError("moco_b200 shuffle: channels_last needs an [N, C, H, W] batch")
        n, C, H, W = x.shape
        _check_nhwc_shape(C, H, W)
        if n and x.stride()[1:] != (H * W, W, 1):          # a channel slice of a wider NCHW batch is read in place
            x = x.contiguous()
        img_stride = x.stride(0) if n else C * H * W
        if s2d:
            # channels_last="s2d": the rows that cross NVLink are already in the space-to-depth layout the stem reads
            _check_s2d_shape(C, H, W)
            R, Q = H // 2 + 3, W // 2 + 3
            row_bytes = R * Q * 16 * 2
            out = torch.empty((src_rows.shape[0], 16, R, Q), dtype=torch.bfloat16, device=x.device,
                              memory_format=torch.channels_last)
            if self.world == 1:
                _lib.check(lib.moco_crop_s2d_bf16(x.data_ptr(), _lib.dtype_code(x), img_stride, src_rows.data_ptr(),
                                                  out.data_ptr(), src_rows.shape[0], H, W, _lib.cur_stream()),
                           "moco_crop_s2d_bf16")
                return out
            buf = self._staging(kind + "_s2d", n * row_bytes)
            _lib.check(lib.moco_crop_s2d_bf16(x.data_ptr(), _lib.dtype_code(x), img_stride, None, buf.local, n, H, W,
                                              _lib.cur_stream()), "moco_crop_s2d_bf16")
            self._pull(buf.table, n, src_rows, row_bytes, out.data_ptr(), synced=True)
            return out
        row_bytes = C * H * W * 2
        if row_bytes % 16 != 0:
            raise ValueError(f"moco_b200 shuffle: row size {row_bytes} B is not a multiple of 16")
        out = torch.empty((src_rows.shape[0], C, H, W), dtype=torch.bfloat16, device=x.device,
                          memory_format=torch.channels_last)
        if self.world == 1:
            # one GPU: the permutation is just the address computation of the crop / cast / layout pass -- ONE kernel
            _lib.check(lib.moco_crop_gather_nhwc_bf16(x.data_ptr(), _lib.dtype_code(x), img_stride, src_rows.data_ptr(),
                                                      out.data_ptr(), src_rows.shape[0], C, H * W, _lib.cur_stream()),
                       "moco_crop_gather_nhwc_bf16")
            return out
        buf = self._staging(kind + "_nhwc", n * row_bytes)
        _lib.check(lib.moco_crop_to_nhwc_bf16(x.data_ptr(), _lib.dtype_code(x), img_stride, buf.local, n, C, H * W,
                                              _lib.cur_stream()), "moco_crop_to_nhwc_bf16")
        self._pull(buf.table, n, src_rows, row_bytes, out.data_ptr(), synced=True)     # publish + ONE pull kernel
        return out


def _check_nhwc_shape(C: int, H: int, W: int) -> None:
    if C > 4 or (H * W) % 8 != 0:
        raise ValueError(f"moco_b200: the fused bf16/NHWC image path needs C <= 4 and H*W % 8 == 0 (got C={C}, H*W={H * W})")


def _check_s2d_shape(C: int, H: int, W: int) -> None:
    if C != 3 or H % 2 or W % 2:
        raise ValueError(f"moco_b200: the space-to-depth input path needs 3 channels and even H, W (got {C}, {H}, {W})")


def crop_to_s2d_bf16(x: torch.Tensor) -> torch.Tensor:
    """[N, 3, H, W] fp32/bf16 (possibly one crop of the 6-channel batch, train.py:250) -> bf16 [N, 16, H/2+3, W/2+3]
    in ``channels_last`` storage: the space-to-depth layout :class:`moco_b200.encoders.StemConv` convolves with a
    4x4 / stride 1 kernel (``moco_crop_s2d_bf16``)."""
    lib = _lib.load()
    _lib.require_cuda(x)
    if x.dim() != 4:
        raise ValueError("crop_to_s2d_bf16: expected [N, 3, H, W]")
    n, C, H, W = x.shape
    _check_s2d_shape(C, H, W)
    if n and x.stride()[1:] != (H * W, W, 1):
        x = x.contiguous()
    out = torch.empty((n, 16, H // 2 + 3, W // 2 + 3), dtype=torch.bfloat16, device=x.device,
                      memory_format=torch.channels_last)
    with torch.cuda.device(x.device):
        _lib.check(lib.moco_crop_s2d_bf16(x.data_ptr(), _lib.dtype_code(x), x.stride(0) if n else C * H * W, None,
                                          out.data_ptr(), n, H, W, _lib.cur_stream()), "moco_crop_s2d_bf16")
    return out


def crop_to_channels_last_bf16(x: torch.Tensor) -> torch.Tensor:
    """[N, C, H, W] fp32/bf16 (possibly a channel slice of a wider NCHW batch, e.g. one crop of the reference's
    6-channel input, train.py:250) -> bf16 tensor of the same shape in ``channels_last`` storage, one kernel
    (``moco_crop_to_nhwc_bf16``).  Bit-identical to ``x.to(torch.bfloat16).contiguous(memory_format=channels_last)``."""
    lib = _lib.load()
    _lib.require_cuda(x)
    if x.dim() != 4:
        raise ValueError("crop_to_channels_last_bf16: expected [N, C, H, W]")
    n, C, H, W = x.shape
    _check_nhwc_shape(C, H, W)
    if n and x.stride()[1:] != (H * W, W, 1):
        x = x.contiguous()
    out = torch.empty((n, C, H, W), dtype=torch.bfloat16, device=x.device, memory_format=torch.channels_last)
    with torch.cuda.device(x.device):
        _lib.check(lib.moco_crop_to_nhwc_bf16(x.data_ptr(), _lib.dtype_code(x), x.stride(0) if n else C * H * W,
                                              out.data_ptr(), n, C, H * W, _lib.cur_stream()), "moco_crop_to_nhwc_bf16")
    return out


# ---------------------------------------------------------------------------
# reference API
# ---------------------------------------------------------------------------
def dist_collect(x):
    """collect all tensor from all GPUs (util.py:47-58): [mini_batch, ...] -> [mini_batch * W, ...],
    rank-major.  Implemented as a P2P pull of every row (identity permutation)."""
    rank, world = _world()
    if world == 1:
        return x.contiguous().clone()
    n = x.shape[0]
    rows = torch.arange(n * world, dtype=torch.long, device=x.device)
    return ShuffleContext.get().gather("collect", x, rows)


class DistributedShufle:
    @staticmethod
    def forward_shuffle(x, epoch, cast_dtype=None, channels_last=False):
        """forward shuffle, return shuffled batch of x from all processes (util.py:69-79).
        epoch is used as manual seed to make sure the shuffle id in all process is same.
        cast_dtype / channels_last: optional extensions, see ShuffleContext.gather (channels_last="s2d": bf16
        space-to-depth rows for encoders.StemConv)."""
        rank, world = _world()
        forward_inds, backward_inds = DistributedShufle.get_shuffle_ids(x.shape[0] * world, epoch, x.device)
        forward_inds_local = DistributedShufle.get_local_id(forward_inds)
        return ShuffleContext.get().gather("fwd", x, forward_inds_local, cast_dtype, channels_last), backward_inds

    @staticmethod
    def backward_shuffle(x, backward_inds, return_local=True):
        """backward shuffle, return data which have been shuffled back (util.py:81-93).
        x is the shared data, should be local data.  if return_local, only return the local batch
        data of x; otherwise, return collected all data on all process."""
        x_all = ShuffleContext.get().gather("bwd", x, backward_inds)      # rank-major original order
        if return_local:
            rank, world = _world()
            n = x.shape[0]
            return x_all, x_all[rank * n:(rank + 1) * n]
        return x_all

    @staticmethod
    def get_local_id(ids):
        rank, world = _world()
        return ids.chunk(world)[rank]

    @staticmethod
    def get_shuffle_ids(bsz, epoch, device=None):
        """generate shuffle ids for ShuffleBN (util.py:99-111); cached per (bsz, epoch, device) --
        the reference recomputes the same permutation (and three H2D copies) every step."""
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device())
        key = (bsz, epoch, str(device))
        hit = _IDS_CACHE.get(key)
        if hit is None:
            if len(_IDS_CACHE) > 64:
                _IDS_CACHE.clear()
            f, b = shuffle_ids_cpu(bsz, epoch)
            hit = _IDS_CACHE[key] = (f.to(device), b.to(device))
        return hit


def set_bn_train(model):
    """key encoder in eval() with BatchNorm layers in train() (util.py:114-121)."""
    def set_bn_train_helper(m):
        if m.__class__.__name__.find('BatchNorm') != -1:
            m.train()

    model.eval()
    model.apply(set_bn_train_helper)


class _EmaPlan:
    """Device-side description of one (model, model_ema) pair for ``moco_ema_update``: an int64 [n, 3] table of
    {p_ema ptr, p ptr, n_elems} and the int32 chunk prefix.  Walking ``parameters()`` of a ResNet-50 twice costs
    ~0.3 ms of host time -- six times the kernel -- so the plan keeps weak references to the Parameter objects
    and re-validates them per call (object still alive, storage not moved); anything else rebuilds the plan."""

    def __init__(self, model, model_ema):
        import weakref
        ps, pes = list(model.parameters()), list(model_ema.parameters())
        if len(ps) != len(pes):
            raise RuntimeError("moco_b200.util.moment_update: model and model_ema have different parameter counts")
        for p, pe in zip(ps, pes):
            if not (pe.is_cuda and p.is_cuda and pe.device == p.device):
                raise RuntimeError("moco_b200.util.moment_update: parameters must live on one CUDA device "
                                   "(there is no CPU fallback)")
            # element i of p must pair with element i of p_ema in STORAGE order: equal strides + dense storage
            # (plain contiguous, or channels_last conv weights as the bf16/NHWC encoders keep them)
            dense = pe.is_contiguous() or (pe.dim() == 4 and pe.is_contiguous(memory_format=torch.channels_last))
            if pe.dtype != torch.float32 or p.dtype != torch.float32 or pe.shape != p.shape \
                    or pe.stride() != p.stride() or not dense:
                raise RuntimeError("moco_b200.util.moment_update: fp32 parameter pairs of equal shape, equal strides "
                                   "and dense storage required")
        self.model_ref = weakref.ref(model)
        self.refs = [weakref.ref(t) for pair in zip(pes, ps) for t in pair]
        self.ptrs = [t.data_ptr() for pair in zip(pes, ps) for t in pair]
        self.n_segs = len(ps)
        self.device = pes[0].device if pes else None
        if not pes:
            return
        chunk = _lib.load().moco_ema_chunk_elems()
        prefix = [0]
        for pe in pes:
            prefix.append(prefix[-1] + (pe.numel() + chunk - 1) // chunk)
        self.n_chunks = prefix[-1]
        table = [(pe.data_ptr(), p.data_ptr(), pe.numel()) for pe, p in zip(pes, ps)]
        self.segs = torch.tensor(table, dtype=torch.int64).reshape(-1, 3).to(self.device)
        self.prefix = torch.tensor(prefix, dtype=torch.int32).to(self.device)

    def valid_for(self, model) -> bool:
        if self.model_ref() is not model:
            return False
        for ref, ptr in zip(self.refs, self.ptrs):
            t = ref()
            if t is None or t.data_ptr() != ptr:
                return False
        return True


@torch.no_grad()
def moment_update(model, model_ema, m):
    """model_ema = m * model_ema + (1 - m) model (util.py:124-127; train.py:133 with m = 0, train.py:277 every
    step) -- one multi-tensor kernel launch (``moco_ema_update``) instead of 2 x #params tiny ones; per element
    fma(1 - m, p, rn(p_ema * m)), bit-exact with the reference's ``mul_(m).add_(1 - m, p)``.

    The parameter walk is cached per (model, model_ema) pair; replacing a Parameter object or moving its storage
    is detected and rebuilds the plan (adding/removing parameters in place is not -- delete
    ``model_ema._moco_ema_plan`` after such surgery)."""
    plan = model_ema.__dict__.get("_moco_ema_plan")
    if plan is None or not plan.valid_for(model):
        plan = _EmaPlan(model, model_ema)
        model_ema.__dict__["_moco_ema_plan"] = plan
    if plan.n_segs == 0:
        return
    lib = _lib.load()
    with torch.cuda.device(plan.device):
        rc = lib.moco_ema_update(plan.segs.data_ptr(), plan.prefix.data_ptr(), plan.n_segs, plan.n_chunks,
                                 float(m), float(1 - m), torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "moco_ema_update")
