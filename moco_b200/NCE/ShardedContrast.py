"""ShardedMemoryMoCo -- MemoryMoCo with the queue partitioned across ranks (BASELINE configs[3]).

Same math as ``moco/NCE/Contrast.py`` (bl0/moco) for a queue of K rows, but rank r stores only ring
slots [r*K/W, (r+1)*K/W): 1/W of the memory and of the HBM bytes per step.  Every rank scores ALL W*N
queries of the step against its shard on the tensor-core kernels (one sweep); three small exchanges stitch
the softmax together -- the step's queries, one (max, sum) pair per query and shard, and the [W*N, C]
partial gradients.  None of them is an NCCL collective: each rank PUBLISHES into a peer-mapped staging
buffer (the kernels write their outputs straight into it), a stream-ordered signal barrier follows, and
the consumers PULL over NVLink -- the same mechanism as ShuffleBN (``moco_b200/util.py``); the partial
gradients are summed by the kernel that finishes dq while it reads the W peers
(``moco_nce_shard_dq_finish_peers``), so no reduce_scatter either.  The only key exchange is ``k_all``,
which ShuffleBN's un-shuffle already produced.  See ``include/moco_b200.h`` (moco_nce_shard_*).
"""
from __future__ import annotations

import ctypes
import math

import torch
import torch.distributed as dist
from torch import nn

from .. import _lib
from .Contrast import _aligned16


def _world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


class _Prof:
    """Optional CUDA-event brackets around the stages of one head evaluation (bench.py's `sharded.parts_us`)."""

    def __init__(self, sink):
        self.sink = sink

    def __call__(self, name):
        return _ProfSpan(self.sink, name)


class _ProfSpan:
    def __init__(self, sink, name):
        self.sink, self.name = sink, name

    def __enter__(self):
        if self.sink is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()

    def __exit__(self, *exc):
        if self.sink is not None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            self.sink.append((self.name, self.e0, e1))


class _ShardedNCE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, k_all, mod):
        from ..util import ShuffleContext
        lib = _lib.load()
        rank, world = _world()
        ctx.set_materialize_grads(False)
        _lib.require_cuda(q, k, k_all, mod.memory)
        q_d = q.detach().contiguous()
        k_d = k.detach().to(q_d.dtype).contiguous()
        k_all = k_all.detach().to(q_d.dtype).contiguous()
        if q_d.dim() != 2 or q_d.shape != k_d.shape or q_d.shape[1] != mod.memory.shape[1]:
            raise ValueError(f"ShardedMemoryMoCo: q {tuple(q_d.shape)} / k {tuple(k_d.shape)} do not match the shard "
                             f"{tuple(mod.memory.shape)}")
        N, C = q_d.shape
        Nq = N * world
        if k_all.shape != (Nq, C):
            raise ValueError(f"ShardedMemoryMoCo: k_all is {tuple(k_all.shape)}, expected ({Nq}, {C})")
        dev = q_d.device
        prof = _Prof(mod.profile)
        sctx = ShuffleContext.get() if world > 1 else None
        with prof("q_exchange_us"):
            if world > 1:
                rows = mod._arange(Nq, dev)
                q_all = sctx.gather("shard_q", q_d, rows)                       # rank-major, like k_all
            else:
                q_all = q_d
        shard = mod._queue_bf16()
        Ks = shard.shape[0]
        ws, ws_ptr, ws_bytes = mod._workspace(Nq, C, dev)
        f32 = dict(dtype=torch.float32, device=dev)
        dt = _lib.dtype_code(q_all)
        stream = _lib.cur_stream()
        inv_T = 1.0 / mod.temperature
        # loss statistics AND the unnormalised gradient partials from one sweep over the shard when a gradient is
        # wanted and the temperature allows it (same policy as moco_nce_fwd, include/moco_b200.h)
        flags = mod.kernel_flags
        if (q.requires_grad and not (flags & (_lib.NCE_TWO_PASS | _lib.NCE_ONE_PASS))
                and inv_T <= _lib.ONE_PASS_MAX_INV_T):
            flags |= _lib.NCE_ONE_PASS
        if not q.requires_grad:
            flags &= ~_lib.NCE_ONE_PASS
        # (max, sum) per query: written straight into the peer-visible staging buffer
        if world > 1:
            ms_buf = sctx._staging("shard_ms", Nq * 8)
            ms = ms_buf.tensor((Nq, 2), torch.float32)
        else:
            ms = torch.empty(Nq, 2, **f32)
        with prof("shard_sweep_us"):
            _lib.check(lib.moco_nce_shard_stats(q_all.data_ptr(), k_all.data_ptr(), dt, shard.data_ptr(), Nq, C, Ks, inv_T,
                                                ms.data_ptr(), ws_ptr, ws_bytes, flags, stream),
                       "moco_nce_shard_stats")
        with prof("stats_exchange_us"):
            if world > 1:
                # pull every rank's [Nq] pairs as 512-byte rows (one warp each); the "published" event rides in the
                # same kernel (moco_shuffle_gather_sync)
                ms_all = torch.empty(world, Nq, 2, **f32)
                if (Nq * 8) % 512 == 0:
                    rpr = Nq * 8 // 512
                    sctx._pull(ms_buf.table, rpr, mod._arange(rpr * world, dev), 512, ms_all.data_ptr(), synced=True)
                else:                                                             # odd sizes: one row per rank
                    sctx._pull(ms_buf.table, 1, mod._arange(world, dev), Nq * 8, ms_all.data_ptr(), synced=True)
            else:
                ms_all = ms
        lse, loss_rows, prob_rows = (torch.empty(Nq, **f32) for _ in range(3))
        loss_prob_all = torch.empty(2, **f32)
        with prof("merge_us"):
            _lib.check(lib.moco_nce_shard_merge(ms_all.data_ptr(), world, Nq, C, inv_T, lse.data_ptr(), loss_rows.data_ptr(),
                                                prob_rows.data_ptr(), loss_prob_all.data_ptr(), ws_ptr, ws_bytes, stream),
                       "moco_nce_shard_merge")
            own = slice(rank * N, (rank + 1) * N)
            loss = loss_rows[own].mean()          # this rank's loss is the mean over ITS rows (train.py:263)
            prob = prob_rows[own].mean()
        ctx.dq = None
        if q.requires_grad:
            if world > 1:
                o_buf = sctx._staging("shard_o", Nq * C * 4)
                o_part = o_buf.tensor((Nq, C), torch.float32)
            else:
                o_part = torch.empty(Nq, C, **f32)
            with prof("dq_partial_us"):
                _lib.check(lib.moco_nce_shard_dq(q_all.data_ptr(), dt, shard.data_ptr(), lse.data_ptr(), Nq, C, Ks, inv_T,
                                                 o_part.data_ptr(), ws_ptr, ws_bytes, flags, stream),
                           "moco_nce_shard_dq")
            dq = torch.empty(N, C, **f32)
            prob_own = prob_rows[own]
            with prof("grad_exchange_us"):
                if world > 1:
                    sctx.barrier()
                    _lib.check(lib.moco_nce_shard_dq_finish_peers(o_buf.table, world, rank, k_d.data_ptr(),
                                                                  _lib.dtype_code(k_d), prob_own.data_ptr(), N, C, inv_T,
                                                                  dq.data_ptr(), stream),
                               "moco_nce_shard_dq_finish_peers")
                else:
                    _lib.check(lib.moco_nce_shard_dq_finish(o_part.data_ptr(), k_d.data_ptr(), _lib.dtype_code(k_d),
                                                            prob_own.data_ptr(), N, C, inv_T, dq.data_ptr(), stream),
                               "moco_nce_shard_dq_finish")
            ctx.dq = dq
        ctx.q_dtype = q.dtype
        ctx.mark_non_differentiable(prob)
        return loss, prob

    @staticmethod
    def backward(ctx, g_loss, g_prob):
        if ctx.dq is None or g_loss is None:
            return None, None, None, None
        return (ctx.dq * g_loss).to(ctx.q_dtype), None, None, None


class ShardedMemoryMoCo(nn.Module):
    """Queue of `queue_size` rows split evenly over the default process group ("block" layout: ring slot g
    lives on rank g // (K/W) at local row g % (K/W)).  `forward_loss(q, k, k_all) -> (loss, prob)`.

    Checkpoint format (train.py:145,163): ``state_dict()`` returns the FULL ``[K, C]`` fp32 ``memory`` -- the same
    keys and shapes as ``MemoryMoCo`` and the reference -- on whichever rank calls it (the reference saves on rank
    0 only, train.py:226-228): the shards live in peer-mapped memory, so the saving rank pulls the other ranks'
    rows over NVLink without their participation.  ``load_state_dict`` accepts a full ``[K, C]`` queue (keeps this
    rank's block) or a bare shard.  ``persist_index=True`` parks the ring position in ``params`` exactly like
    ``MemoryMoCo(persist_index=True)``."""

    def __init__(self, feature_dim, queue_size, temperature=0.07, persist_index=False):
        super().__init__()
        rank, world = _world()
        if queue_size % world != 0:
            raise ValueError(f"queue_size {queue_size} is not divisible by the world size {world}")
        self.queue_size = queue_size
        self.temperature = temperature
        self.index = 0
        self.kernel_flags = _lib.NCE_AUTO
        self.persist_index = bool(persist_index)
        self.profile = None           # set to a list to collect (stage, start_event, stop_event) triples
        self.shard_rows = queue_size // world
        self.shard_row0 = rank * self.shard_rows
        self.register_buffer('params', torch.tensor([-1]))
        # identical initial queue on every rank (same global RNG stream as the reference, Contrast.py:16-17),
        # of which this rank keeps its block
        stdv = 1. / math.sqrt(feature_dim / 3)
        full = torch.rand(queue_size, feature_dim).mul_(2 * stdv).add_(-stdv)
        self.register_buffer('memory', full[self.shard_row0:self.shard_row0 + self.shard_rows].clone())
        self.register_buffer('memory_bf16', torch.empty(0, dtype=torch.bfloat16), persistent=False)
        self._bf16_src = None
        self._ws = {}
        self._ar = {}
        self._peer_mem = None         # _PeerBuffer holding `memory` once share_memory_across_ranks() ran
        self.register_load_state_dict_post_hook(lambda m, keys: m._after_load())

    def _apply(self, fn, *a, **kw):
        if self._peer_mem is not None:
            raise RuntimeError("ShardedMemoryMoCo: the shard lives in peer-mapped memory and cannot be moved or "
                               "converted after the first step; call .to(device) before training")
        out = super()._apply(fn, *a, **kw)
        self._bf16_src = None
        self._ws = {}
        self._ar = {}
        return out

    def _arange(self, n, dev):
        t = self._ar.get((n, dev))
        if t is None:
            t = self._ar[(n, dev)] = torch.arange(n, dtype=torch.long, device=dev)
        return t

    # -- peer-visible shard (checkpointing without a collective) ---------------------------------------------
    @torch.no_grad()
    def share_memory_across_ranks(self):
        """COLLECTIVE (every rank, same point): move the fp32 shard into a CUDA-IPC mapped buffer every peer can read.
        Called automatically by the first forward_loss."""
        rank, world = _world()
        if world == 1 or self._peer_mem is not None:
            return
        from ..util import _PeerBuffer
        _lib.require_cuda(self.memory)
        self._check_buffers()
        buf = _PeerBuffer(self.memory.numel() * 4, rank, world)
        view = buf.tensor(tuple(self.memory.shape), torch.float32)
        view.copy_(self.memory)
        self.memory = view            # same registered buffer name, now backed by the peer-mapped allocation
        self._peer_mem = buf
        self._bf16_src = None

    @torch.no_grad()
    def full_memory(self):
        """[K, C] fp32 queue assembled from every rank's shard (checkpoint-compatible with MemoryMoCo's `memory`).
        Not a collective once the shards are peer-mapped: a single rank may call it."""
        rank, world = _world()
        if world == 1:
            return self.memory.clone()
        if self._peer_mem is None:
            raise RuntimeError("ShardedMemoryMoCo: shards are not peer-mapped yet (no step has run); call "
                               "share_memory_across_ranks() on every rank first")
        lib = _lib.load()
        C = self.memory.shape[1]
        out = torch.empty(self.queue_size, C, dtype=torch.float32, device=self.memory.device)
        rows = self._arange(self.queue_size, self.memory.device)
        torch.cuda.current_stream().synchronize()
        _lib.check(lib.moco_shuffle_gather(self._peer_mem.table, world, self.shard_rows, rows.data_ptr(), self.queue_size,
                                           C * 4, out.data_ptr(), 0, _lib.cur_stream()), "moco_shuffle_gather")
        return out

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        if self.persist_index:
            self.params.fill_(int(self.index))
        super()._save_to_state_dict(destination, prefix, keep_vars)
        if _world()[1] > 1:
            destination[prefix + 'memory'] = self.full_memory()

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        key = prefix + 'memory'
        mem = state_dict.get(key)
        if mem is not None and mem.dim() == 2 and mem.shape[0] == self.queue_size and self.shard_rows != self.queue_size:
            state_dict = dict(state_dict)             # a full [K, C] queue (MemoryMoCo / reference / our own save)
            state_dict[key] = mem[self.shard_row0:self.shard_row0 + self.shard_rows]
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    def _after_load(self):
        self._bf16_src = None
        if self.persist_index:
            saved = int(self.params.item())
            self.index = saved % self.queue_size if saved >= 0 else 0

    # -- bf16 working shard ----------------------------------------------------------------------------------
    def _check_buffers(self):
        mem = self.memory
        if mem.dtype != torch.float32 or not mem.is_contiguous() or mem.dim() != 2 or mem.shape[0] != self.shard_rows:
            raise RuntimeError(f"ShardedMemoryMoCo: `memory` must stay a contiguous float32 [K/W, C] buffer "
                               f"(got {mem.dtype}, shape {tuple(mem.shape)})")

    def _queue_bf16(self):
        mem = self.memory
        _lib.require_cuda(mem)
        self._check_buffers()
        tag = (mem.data_ptr(), mem._version)
        if self._bf16_src != tag or self.memory_bf16.shape != mem.shape or self.memory_bf16.device != mem.device:
            self.memory_bf16 = torch.empty(mem.shape, dtype=torch.bfloat16, device=mem.device)
            lib = _lib.load()
            _lib.check(lib.moco_f32_to_bf16(mem.data_ptr(), self.memory_bf16.data_ptr(), mem.numel(), _lib.cur_stream()),
                       "moco_f32_to_bf16")
            self._bf16_src = tag
        return self.memory_bf16

    def _workspace(self, Nq, C, dev):
        key = (Nq, C, dev)
        hit = self._ws.get(key)
        if hit is None:
            lib = _lib.load()
            nbytes = int(lib.moco_nce_workspace_bytes(Nq, C, self.shard_rows))
            t = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
            hit = self._ws[key] = (t, t.data_ptr() + (-t.data_ptr()) % 256, nbytes)
        return hit

    @torch.no_grad()
    def enqueue(self, k_all):
        lib = _lib.load()
        _lib.require_cuda(k_all)
        k_all = _aligned16(k_all.detach().contiguous())
        if k_all.dim() != 2 or k_all.shape[1] != self.memory.shape[1] or k_all.device != self.memory.device:
            raise ValueError(f"ShardedMemoryMoCo.enqueue: k_all {tuple(k_all.shape)} on {k_all.device} does not match "
                             f"the shard {tuple(self.memory.shape)} on {self.memory.device}")
        if k_all.shape[0] > self.queue_size:
            raise ValueError(f"ShardedMemoryMoCo.enqueue: {k_all.shape[0]} keys > queue_size {self.queue_size}")
        n_all, C = k_all.shape
        shard = self._queue_bf16()
        _lib.check(lib.moco_queue_enqueue_shard(shard.data_ptr(), self.memory.data_ptr(), k_all.data_ptr(),
                                                _lib.dtype_code(k_all), n_all, C, self.queue_size, self.index,
                                                self.shard_row0, self.shard_rows, _lib.cur_stream()),
                   "moco_queue_enqueue_shard")
        self._bf16_src = (self.memory.data_ptr(), self.memory._version)
        self.index = (self.index + n_all) % self.queue_size

    def forward_loss(self, q, k, k_all):
        self.share_memory_across_ranks()
        loss, prob = _ShardedNCE.apply(q, k.detach(), k_all, self)
        self.enqueue(k_all)
        return loss, prob
