"""Minimal MoCo pre-training driver on the H100-native hot path -- what bl0/moco's ``train.py`` main loop
(train.py:231-293) looks like once ``MemoryMoCo`` / ``DistributedShufle`` / ``moment_update`` come from
``moco_b200`` (INTEGRATION.md).  Not a port of the reference's control plane (logging, LR schedule, dataset,
checkpoint rotation are out of scope, SURVEY.md §8): synthetic images, SGD, N steps.

Launch compatibility (SURVEY.md §8b): the reference only understands ``--local_rank`` (train.py:81), which
``torch.distributed.launch`` on torch >= 2.0 no longer passes (``--local-rank``) and ``torchrun`` never did
(``$LOCAL_RANK``).  This entry point accepts all three:

    python examples/train_moco.py --steps 20                                            # 1 GPU
    python examples/train_moco.py --data-dir /data/imagenet --steps 20                  # real images (train/)
    torchrun --nproc-per-node 8 --master-addr 127.0.0.1 examples/train_moco.py --steps 20
"""
import argparse
import os


def parse_args(argv=None):
    ap = argparse.ArgumentParser("moco_b200 example trainer")
    ap.add_argument("--local_rank", "--local-rank", dest="local_rank", type=int,
                    default=int(os.environ.get("LOCAL_RANK", 0)), help="GPU of this process (default: $LOCAL_RANK)")
    ap.add_argument("--arch", default="resnet50", choices=["resnet18", "resnet34", "resnet50"])
    ap.add_argument("--batch-size", type=int, default=256, help="per GPU (train.py: --batch-size)")
    ap.add_argument("--nce-k", type=int, default=16384)
    ap.add_argument("--nce-t", type=float, default=0.07)
    ap.add_argument("--alpha", type=float, default=0.999, help="EMA momentum of the key encoder")
    ap.add_argument("--base-lr", type=float, default=0.03)
    ap.add_argument("--momentum", type=float, default=0.9)
    ap.add_argument("--weight-decay", type=float, default=1e-4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--epoch", type=int, default=1, help="ShuffleBN seed (train.py:258 uses the epoch number)")
    ap.add_argument("--resume", default="", help="checkpoint written by --save or by the reference (either key naming)")
    ap.add_argument("--save", default="")
    ap.add_argument("--persist-index", action="store_true", help="keep the queue write position across resume")
    ap.add_argument("--fuse-normalize", action="store_true",
                    help="encoders return the raw fc output; L2 normalisation (resnet.py:24-33) runs inside the head kernels")
    ap.add_argument("--graph-tail", action="store_true",
                    help="single GPU: replay everything after the key encoder from one CUDA graph (device-side ring index)")
    ap.add_argument("--data-dir", default="",
                    help="ImageFolder root with train/ (train.py:94); decoded by the workers, augmented on the GPU "
                         "(moco_b200/augment.py).  Without it the inputs are synthetic.")
    ap.add_argument("--crop", type=float, default=0.08, help="minimum crop scale (train.py: --crop)")
    ap.add_argument("--aug", default="CJ", choices=["NULL", "CJ"], help="train.py: --aug")
    ap.add_argument("--num-workers", type=int, default=4, help="DataLoader workers per GPU (train.py: --num-workers)")
    return ap.parse_args(argv)


def make_loader(args, world):
    """train.py:92-125 with the pixel work moved to the GPU: the workers decode and draw the crop parameters only."""
    import torch
    from moco_b200.augment import ImageFolderTwoCrop
    dataset = ImageFolderTwoCrop(os.path.join(args.data_dir, "train"), scale=(args.crop, 1.0), aug=args.aug)
    sampler = torch.utils.data.distributed.DistributedSampler(dataset, drop_last=True) if world > 1 else None
    return torch.utils.data.DataLoader(dataset, batch_size=args.batch_size, shuffle=sampler is None,
                                       num_workers=args.num_workers, pin_memory=True, sampler=sampler,
                                       drop_last=True, collate_fn=ImageFolderTwoCrop.collate_fn,
                                       persistent_workers=args.num_workers > 0)


def main(argv=None):
    args = parse_args(argv)
    import torch
    import torch.distributed as dist
    from moco_b200 import encoders
    from moco_b200.encoders import from_reference_state_dict
    from moco_b200.NCE import MemoryMoCo
    from moco_b200.train_step import MoCoStep
    from moco_b200.util import moment_update

    world = int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(args.local_rank)
    dev = torch.device("cuda", args.local_rank)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)                                   # train.py:300
    rank = dist.get_rank() if world > 1 else 0

    torch.manual_seed(0)
    ctor = getattr(encoders, args.arch)
    model = ctor(low_dim=128).to(dev).to(memory_format=torch.channels_last)
    model_ema = ctor(low_dim=128).to(dev).to(memory_format=torch.channels_last)
    moment_update(model, model_ema, 0)                                                    # train.py:133
    contrast = MemoryMoCo(128, args.nce_k, args.nce_t, persist_index=args.persist_index,
                          device_index=args.graph_tail).to(dev)                          # train.py:181
    opt = torch.optim.SGD(model.parameters(), lr=args.base_lr * args.batch_size * world / 256,
                          momentum=args.momentum, weight_decay=args.weight_decay)        # train.py:183-187
    if args.resume:
        ckpt = torch.load(args.resume, map_location="cpu")                               # train.py:157-166
        model.load_state_dict(from_reference_state_dict(ckpt["model"]))
        model_ema.load_state_dict(from_reference_state_dict(ckpt["model_ema"]))
        contrast.load_state_dict(ckpt["contrast"])
        opt.load_state_dict(ckpt["optimizer"])
    if world > 1:
        model = torch.nn.parallel.DistributedDataParallel(model, device_ids=[args.local_rank],
                                                          broadcast_buffers=False)     # train.py:198
    step = MoCoStep(model, model_ema, contrast, opt, alpha=args.alpha, channels_last=True,
                    fuse_normalize=args.fuse_normalize, graph_tail=args.graph_tail)

    gen = torch.Generator(device=dev).manual_seed(1234 + rank)
    batches = None
    if args.data_dir:
        from moco_b200.augment import augment_two_crop
        loader = make_loader(args, world)
        batches = _cycle(loader)
    for it in range(args.steps):
        if batches is not None:
            inputs = augment_two_crop(next(batches))                                     # replaces train.py:253-254
        else:
            inputs = torch.randn(args.batch_size, 6, 224, 224, device=dev, generator=gen)    # dataset.py:31-33 layout
        x1, x2 = torch.split(inputs, [3, 3], dim=1)                                      # train.py:250
        loss, prob = step(x1, x2, args.epoch)
        if rank == 0 and (it % 10 == 0 or it == args.steps - 1):
            print(f"step {it:4d}  loss {loss.item():.4f}  prob {prob.item():.5f}", flush=True)
    if args.save and rank == 0:
        net = model.module if hasattr(model, "module") else model
        torch.save({"model": net.state_dict(), "model_ema": model_ema.state_dict(), "contrast": contrast.state_dict(),
                    "optimizer": opt.state_dict(), "epoch": args.epoch}, args.save)     # train.py:141-150
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def _cycle(loader):
    epoch = 0
    while True:
        if getattr(loader, "sampler", None) is not None and hasattr(loader.sampler, "set_epoch"):
            loader.sampler.set_epoch(epoch)                                              # train.py:213
        yield from loader
        epoch += 1


if __name__ == "__main__":
    main()
