"""SURVEY.md §8(d): "the reference PyTorch path on the same GPU as the primary beat-this baseline for every
kernel".  Times, on one GPU with CUDA events, the post-encoder head (a7-a11: logits + loss + prob + backward to
q + enqueue) and the EMA update (f1) two ways:

  * `torch`  : the reference's sequence of PyTorch library calls restated here op for op
               (Contrast.py:20-34, NCECriterion.py:11-13, train.py:264,273, util.py:124-127) -- fp32 as the
               reference runs it without Apex, and with a bf16 mm (what Apex O1 / autocast would do);
  * `native` : moco_b200 through the C ABI (MemoryMoCo.forward_loss + backward, util.moment_update).

Prints one JSON line per case.  Measurement tool only; nothing in the product imports it.

    python tools/torch_gpu_baseline.py [c2 c3 c5 ema]
    torchrun --nproc-per-node W tools/torch_gpu_baseline.py shuffle step     # multi-GPU rows (SURVEY 8d, VERDICT r1 #5)

`shuffle`: ShuffleBN as the reference runs it -- W x zeros_like, NCCL all_gather, cat, fancy index (util.py:47-58,
74-79, 88-91) -- restated op for op on the BASELINE batch, beside moco_b200's P2P pull (publish + one kernel).
`step`: the whole reference iteration (train.py:244-283) as its sequence of PyTorch ops on the same GPUs -- fp32
encoders as the reference runs them without Apex, NCCL ShuffleBN, torch.mm head with the queue clone, per-parameter
EMA loop, two .item() syncs -- beside MoCoStep on the same encoder class.
"""
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HEAD = {"c1": (32, 128, 1024), "c2": (256, 128, 16384), "c3": (256, 128, 65536), "c4shard": (2048, 128, 16384),
        "c5": (512, 256, 262144)}
T = 0.07


def time_cuda(fn, iters, warmup=5, flush=None):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    total = 0.0
    for _ in range(iters):
        if flush is not None:
            flush.add_(1)                                    # > L2 (126 MB): evict the queue between iterations
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        total += s.elapsed_time(e)
    return total / iters * 1e3                               # us


class TorchHead:
    """The reference head as PyTorch library calls (op-for-op restatement for timing)."""

    def __init__(self, C, K, mm_dtype):
        self.K, self.index, self.mm_dtype = K, 0, mm_dtype
        stdv = 1.0 / (C / 3) ** 0.5
        self.memory = torch.rand(K, C, device="cuda").mul_(2 * stdv).add_(-stdv)

    def step(self, q, k, k_all):
        k = k.detach()
        l_pos = (q * k).sum(dim=-1, keepdim=True)
        mem = self.memory.clone().detach()
        if self.mm_dtype is torch.float32:
            l_neg = torch.mm(q, mem.transpose(1, 0))
        else:
            l_neg = torch.mm(q.to(self.mm_dtype), mem.to(self.mm_dtype).transpose(1, 0)).float()
        out = torch.cat((l_pos, l_neg), dim=1) / T
        out = out.contiguous()
        with torch.no_grad():
            n_all = k_all.shape[0]
            ids = torch.fmod(torch.arange(n_all, dtype=torch.long) + self.index, self.K).cuda()
            self.memory.index_copy_(0, ids, k_all)
            self.index = (self.index + n_all) % self.K
        label = torch.zeros(out.shape[0], dtype=torch.long, device="cuda")
        loss = F.cross_entropy(out, label)
        prob = F.softmax(out, dim=1)[:, 0].mean()
        loss.backward()
        return loss, prob


def run_head(name):
    from moco_b200.NCE import MemoryMoCo
    N, C, K = HEAD[name]
    torch.manual_seed(0)
    q0 = F.normalize(torch.randn(N, C, device="cuda"), dim=1)
    k = F.normalize(torch.randn(N, C, device="cuda"), dim=1)
    k_all = k.clone()
    flush = torch.zeros(64 << 20, dtype=torch.float32, device="cuda") if K * C * 4 < (200 << 20) else None
    iters = 30 if K <= 65536 else 10
    res = {"case": f"head_{name}", "N": N, "C": C, "K": K, "l2_flush": flush is not None}

    for tag, dt in (("torch_fp32", torch.float32), ("torch_bf16mm", torch.bfloat16)):
        head = TorchHead(C, K, dt)

        def f():
            q = q0.clone().requires_grad_(True)
            head.step(q, k, k_all)
        res[f"{tag}_us"] = round(time_cuda(f, iters, flush=flush), 1)
        del head

    contrast = MemoryMoCo(C, K, T).cuda()

    def g():
        q = q0.clone().requires_grad_(True)
        loss, prob = contrast.forward_loss(q, k, k_all)
        loss.backward()
    res["native_us"] = round(time_cuda(g, iters, flush=flush), 1)
    res["speedup_vs_torch_fp32"] = round(res["torch_fp32_us"] / res["native_us"], 2)
    res["speedup_vs_torch_bf16mm"] = round(res["torch_bf16mm_us"] / res["native_us"], 2)
    print(json.dumps(res), flush=True)


def run_ema(_):
    from moco_b200 import encoders
    from moco_b200.util import moment_update
    model, ema = encoders.resnet50(low_dim=128).cuda(), encoders.resnet50(low_dim=128).cuda()
    n = sum(p.numel() for p in model.parameters())
    flush = torch.zeros(64 << 20, dtype=torch.float32, device="cuda")

    def ref():                                               # util.py:124-127 verbatim semantics
        for p1, p2 in zip(model.parameters(), ema.parameters()):
            p2.data.mul_(0.999).add_(p1.detach().data, alpha=1 - 0.999)

    def foreach():
        pe = [p.data for p in ema.parameters()]
        torch._foreach_mul_(pe, 0.999)
        torch._foreach_add_(pe, [p.detach().data for p in model.parameters()], alpha=1 - 0.999)

    res = {"case": "ema_resnet50", "params": n, "tensors": len(list(model.parameters())), "l2_flush": True}
    res["torch_loop_us"] = round(time_cuda(ref, 20, flush=flush), 1)
    res["torch_foreach_us"] = round(time_cuda(foreach, 20, flush=flush), 1)
    res["native_us"] = round(time_cuda(lambda: moment_update(model, ema, 0.999), 20, flush=flush), 1)
    # the kernel alone (the line above includes the Python-side pointer check of 161 parameter pairs)
    from moco_b200 import _lib
    lib, plan = _lib.load(), ema._moco_ema_plan
    st = torch.cuda.current_stream().cuda_stream

    def kern():
        lib.moco_ema_update(plan.segs.data_ptr(), plan.prefix.data_ptr(), plan.n_segs, plan.n_chunks, 0.999, 1 - 0.999, st)
    res["native_kernel_us"] = round(time_cuda(kern, 20, flush=flush), 1)
    res["native_kernel_GBps"] = round(12.0 * n / (res["native_kernel_us"] * 1e-6) / 1e9, 1)
    res["speedup_vs_torch_loop"] = round(res["torch_loop_us"] / res["native_us"], 2)
    print(json.dumps(res), flush=True)


# ---------------------------------------------------------------- multi-GPU rows (run under torchrun)
def _dist():
    import torch.distributed as dist
    if not dist.is_initialized():
        local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local)
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29533")
        os.environ.setdefault("RANK", "0")
        os.environ.setdefault("WORLD_SIZE", "1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    return dist, dist.get_rank(), dist.get_world_size()


def ref_dist_collect(dist, x):                               # util.py:47-58
    x = x.contiguous()
    out_list = [torch.zeros_like(x, device=x.device, dtype=x.dtype) for _ in range(dist.get_world_size())]
    dist.all_gather(out_list, x)
    return torch.cat(out_list, dim=0)


def time_ranks(dist, fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1) / iters], device="cuda")
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    return float(ms) * 1e3


def run_shuffle(_):
    from moco_b200.util import DistributedShufle
    dist, rank, world = _dist()
    n = 256
    torch.manual_seed(rank)
    x = torch.randn(n, 3, 224, 224, device="cuda")
    feat = torch.randn(n, 128, device="cuda")
    fwd, bwd = DistributedShufle.get_shuffle_ids(n * world, 5, x.device)

    def ref_fwd():                                           # util.py:69-79 (ids cached: the reference recomputes them)
        x_all = ref_dist_collect(dist, x)
        return x_all[fwd.chunk(world)[rank]]

    def ref_bwd():                                           # util.py:81-93
        x_all = ref_dist_collect(dist, feat)
        return x_all[bwd], x_all[bwd.chunk(world)[rank]]
    res = {"case": "shufflebn", "world": world, "rows": n, "image_bytes_fp32": x[0].numel() * 4}
    res["torch_nccl_fwd_fp32_us"] = round(time_ranks(dist, ref_fwd, 10), 1)
    res["torch_nccl_bwd_us"] = round(time_ranks(dist, ref_bwd, 20), 1)
    xb = x.bfloat16()
    res["torch_nccl_fwd_bf16_us"] = round(time_ranks(dist, lambda: ref_dist_collect(dist, xb)[fwd.chunk(world)[rank]], 10), 1)
    res["native_fwd_fp32_us"] = round(time_ranks(dist, lambda: DistributedShufle.forward_shuffle(x, 5), 10), 1)
    res["native_fwd_bf16_nhwc_us"] = round(time_ranks(dist, lambda: DistributedShufle.forward_shuffle(x, 5, channels_last=True), 10), 1)
    res["native_bwd_us"] = round(time_ranks(dist, lambda: DistributedShufle.backward_shuffle(feat, bwd, True), 20), 1)
    # correctness of the comparison itself
    a, b = ref_fwd(), DistributedShufle.forward_shuffle(x, 5)[0]
    res["same_result"] = bool(torch.equal(a, b))
    res["speedup_fwd_fp32"] = round(res["torch_nccl_fwd_fp32_us"] / res["native_fwd_fp32_us"], 2)
    res["speedup_fwd_as_used"] = round(res["torch_nccl_fwd_fp32_us"] / res["native_fwd_bf16_nhwc_us"], 2)
    if rank == 0:
        print(json.dumps(res), flush=True)


def run_step(_):
    """train.py:244-283 as its PyTorch ops (fp32, the reference's default without Apex) vs MoCoStep, same encoder class."""
    from moco_b200 import encoders
    from moco_b200.NCE import MemoryMoCo
    from moco_b200.train_step import MoCoStep
    dist, rank, world = _dist()
    N, C, K = 256, 128, 16384 if world == 1 else 65536
    torch.backends.cudnn.benchmark = True
    torch.manual_seed(0)
    model, ema = encoders.resnet50(low_dim=C).cuda(), encoders.resnet50(low_dim=C).cuda()
    ema.load_state_dict(model.state_dict())
    opt = torch.optim.SGD(model.parameters(), lr=0.03, momentum=0.9, weight_decay=1e-4)
    ddp = torch.nn.parallel.DistributedDataParallel(model, device_ids=[torch.cuda.current_device()], broadcast_buffers=False)
    head = TorchHead(C, K, torch.float32)
    inputs = torch.randn(N, 6, 224, 224, device="cuda")
    ddp.train()
    from moco_b200.util import set_bn_train
    set_bn_train(ema)

    def ref_step():
        x1, x2 = torch.split(inputs, [3, 3], dim=1)
        x1, x2 = x1.contiguous(), x2.contiguous()
        feat_q = ddp(x1)
        with torch.no_grad():
            torch.manual_seed(1)                             # util.py:102: reseeds the global RNG every step
            fwd = torch.randperm(N * world).long().cuda()
            bwd = torch.zeros(N * world).long().cuda()
            bwd.index_copy_(0, fwd, torch.arange(N * world).long().cuda())
            x2s = ref_dist_collect(dist, x2)[fwd.chunk(world)[rank]]
            feat_k = ema(x2s)
            k_all_g = ref_dist_collect(dist, feat_k)
            k_all, k_loc = k_all_g[bwd], k_all_g[bwd.chunk(world)[rank]]
        opt.zero_grad()
        loss, prob = head.step(feat_q, k_loc, k_all)          # includes loss.backward() (train.py:262-273)
        opt.step()
        for p1, p2 in zip(model.parameters(), ema.parameters()):     # util.py:124-127
            p2.data.mul_(0.999).add_(p1.detach().data, alpha=1 - 0.999)
        return loss.item(), prob.item()                      # train.py:280-281
    res = {"case": "full_step", "world": world, "batch_per_gpu": N, "K": K}
    us = time_ranks(dist, ref_step, 8, warmup=3)
    res["torch_reference_ops_fp32_ms"] = round(us / 1e3, 2)
    res["torch_reference_ops_fp32_img_s"] = round(N * world / (us * 1e-6), 1)
    del ddp, head
    torch.cuda.empty_cache()
    model2 = encoders.resnet50(low_dim=C).cuda().to(memory_format=torch.channels_last)
    ema2 = encoders.resnet50(low_dim=C).cuda().to(memory_format=torch.channels_last)
    ema2.load_state_dict(model2.state_dict())
    opt2 = torch.optim.SGD(model2.parameters(), lr=0.03, momentum=0.9, weight_decay=1e-4)
    ddp2 = torch.nn.parallel.DistributedDataParallel(model2, device_ids=[torch.cuda.current_device()], broadcast_buffers=False,
                                                     gradient_as_bucket_view=True, static_graph=True)
    step = MoCoStep(ddp2, ema2, MemoryMoCo(C, K, T).cuda(), opt2, channels_last=True)
    x1, x2 = torch.split(inputs, [3, 3], dim=1)
    us2 = time_ranks(dist, lambda: step(x1, x2, 1), 8, warmup=3)
    res["moco_b200_bf16_ms"] = round(us2 / 1e3, 2)
    res["moco_b200_bf16_img_s"] = round(N * world / (us2 * 1e-6), 1)
    res["speedup"] = round(us / us2, 2)
    if rank == 0:
        print(json.dumps(res), flush=True)


def main():
    assert torch.cuda.is_available()
    names = sys.argv[1:] or ["c2", "c3", "c5", "ema"]
    for n in names:
        {"ema": run_ema, "shuffle": run_shuffle, "step": run_step}.get(n, run_head)(n)
    import torch.distributed as dist
    if dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
