"""MoCo pre-training on the H100-native hot path -- bl0/moco's ``train.py`` (train.py:175-293) once ``MemoryMoCo`` /
``DistributedShufle`` / ``moment_update`` come from ``moco_b200`` (INTEGRATION.md).  Three modes:

* ``--data-dir D`` without ``--steps``: train.py's recipe on the image folder ``D/train``.  Epochs with a
  ``DistributedSampler``, the per-iteration warm-up + cosine / step schedule (``moco_b200.linear_eval.get_scheduler``),
  ShuffleBN seeded by the loop epoch, and every epoch ``current.pth`` (plus ``ckpt_epoch_{e}.pth`` every
  ``--save-freq`` epochs) under ``--output-dir`` in the reference's checkpoint format (``moco_b200.checkpoint``).
  train.py's flags and defaults (batch 128, K = 65536, base lr 0.1, 200 epochs); ``--resume`` takes this format or
  the reference's own ``current.pth``.  Epoch e's crops depend only on ``--rng-seed``, e and the loader
  configuration, so a resumed run trains on the same crops as an uninterrupted one.
* ``--data-dir D --steps N``: N steps on ``D/train``, no schedule.
* no ``--data-dir``: N steps on synthetic images.
The last two take batch 256, K = 16384 and base lr 0.03 by default, and write a checkpoint only with ``--save``.

Launch compatibility (SURVEY.md §8b): the reference only understands ``--local_rank`` (train.py:81), which
``torch.distributed.launch`` on torch >= 2.0 no longer passes (``--local-rank``) and ``torchrun`` never did
(``$LOCAL_RANK``).  This entry point accepts all three:

    python examples/train_moco.py --data-dir /data/imagenet --output-dir ./output               # the recipe, 1 GPU
    torchrun --nproc-per-node 8 examples/train_moco.py --data-dir /data/imagenet --nce-k 65536 --output-dir ./output
    python examples/train_moco.py --steps 20                                                    # synthetic
    python examples/train_moco.py --data-dir /data/imagenet --steps 20                          # real images, 20 steps
"""
import argparse
import os


# train.py's defaults where they differ from those of the step-count modes
RECIPE_DEFAULTS = {"batch_size": 128, "nce_k": 65536, "base_lr": 0.1}
STEPS_DEFAULTS = {"batch_size": 256, "nce_k": 16384, "base_lr": 0.03, "steps": 20}


def parse_args(argv=None):
    """The recipe runs when --data-dir is given and --steps is not; its args have ``steps`` None."""
    ap = argparse.ArgumentParser("moco_b200 example trainer")
    ap.add_argument("--local_rank", "--local-rank", dest="local_rank", type=int,
                    default=int(os.environ.get("LOCAL_RANK", 0)), help="GPU of this process (default: $LOCAL_RANK)")
    ap.add_argument("--arch", default="resnet50", choices=["resnet18", "resnet34", "resnet50"])
    ap.add_argument("--model-width", type=int, default=1, help="width of the ResNet (train.py: --model-width)")
    ap.add_argument("--batch-size", type=int, default=None, help="per GPU (train.py: --batch-size; default 128 in "
                                                                 "the recipe, else 256)")
    ap.add_argument("--nce-k", type=int, default=None, help="queue size (default 65536 in the recipe, else 16384)")
    ap.add_argument("--nce-t", type=float, default=0.07)
    ap.add_argument("--alpha", type=float, default=0.999, help="EMA momentum of the key encoder")
    ap.add_argument("--base-lr", "--base-learning-rate", dest="base_lr", type=float, default=None,
                    help="learning rate at 256 images per step, scaled linearly (default 0.1 in the recipe, else 0.03)")
    ap.add_argument("--momentum", type=float, default=0.9)
    ap.add_argument("--weight-decay", type=float, default=1e-4)
    ap.add_argument("--steps", type=int, default=None, help="run this many steps (default 20 without --data-dir); "
                                                            "with --data-dir and without --steps the recipe runs")
    ap.add_argument("--epoch", type=int, default=1, help="ShuffleBN seed of the step-count modes (the recipe uses "
                                                         "the loop epoch, as train.py:258)")
    ap.add_argument("--resume", default="", help="checkpoint written by this script or by the reference (either key naming)")
    ap.add_argument("--save", default="", help="step-count modes: write a checkpoint here at the end")
    ap.add_argument("--persist-index", action="store_true", help="keep the queue write position across resume")
    ap.add_argument("--fuse-normalize", action="store_true",
                    help="encoders return the raw fc output; L2 normalisation (resnet.py:24-33) runs inside the head kernels")
    ap.add_argument("--graph-tail", action="store_true",
                    help="single GPU: replay everything after the key encoder from one CUDA graph (device-side ring index)")
    ap.add_argument("--data-dir", default="",
                    help="ImageFolder root with train/ (train.py:94); decoded by the workers, augmented on the GPU "
                         "(moco_b200/augment.py).  Without it the inputs are synthetic.")
    ap.add_argument("--crop", type=float, default=0.08, help="minimum crop scale (train.py: --crop)")
    ap.add_argument("--aug", default="CJ", choices=["NULL", "CJ", "V2"],
                    help="train.py: --aug; V2 is MoCo v2's aug-plus (colour jitter 0.8, grayscale after it, Gaussian "
                         "blur 0.5; moco_b200/augment.py)")
    ap.add_argument("--mlp", action="store_true",
                    help="MoCo v2's projection head: fc is Linear(C, C) -> ReLU -> Linear(C, 128)")
    ap.add_argument("--num-workers", type=int, default=4, help="DataLoader workers per GPU (train.py: --num-workers)")
    # the recipe (train.py's flags and defaults)
    ap.add_argument("--epochs", type=int, default=200)
    ap.add_argument("--lr-scheduler", default="cosine", choices=["step", "cosine"])
    ap.add_argument("--warmup-epoch", type=int, default=5)
    ap.add_argument("--warmup-multiplier", type=int, default=100)
    ap.add_argument("--lr-decay-epochs", type=int, default=[120, 160, 200], nargs="+")
    ap.add_argument("--lr-decay-rate", type=float, default=0.1)
    ap.add_argument("--output-dir", default="./output", help="config.json and the checkpoints")
    ap.add_argument("--save-freq", type=int, default=10, help="also keep ckpt_epoch_{e}.pth every this many epochs")
    ap.add_argument("--print-freq", type=int, default=10)
    ap.add_argument("--rng-seed", type=int, default=0, help="seeds the models' initialisation and the crop draws")
    # accepted so that the reference's command lines parse; the step always runs bf16 autocast
    ap.add_argument("--dataset", default="imagenet", choices=["imagenet100", "imagenet"], help="no effect")
    ap.add_argument("--amp-opt-level", default="O0", choices=["O0", "O1", "O2"], help="no effect")
    args = ap.parse_args(argv)
    recipe = bool(args.data_dir) and args.steps is None
    for k, v in (RECIPE_DEFAULTS if recipe else STEPS_DEFAULTS).items():
        if getattr(args, k) is None:
            setattr(args, k, v)
    return args


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


def make_recipe_loader(args, world, rank):
    """train.py:92-125 for the recipe: a DistributedSampler at every world size (train.py:119), drop_last, and
    workers that start afresh every epoch from the loader's own generator, which ``seed_epoch`` re-seeds."""
    import torch
    from moco_b200.augment import ImageFolderTwoCrop
    dataset = ImageFolderTwoCrop(os.path.join(args.data_dir, "train"), scale=(args.crop, 1.0), aug=args.aug)
    sampler = torch.utils.data.distributed.DistributedSampler(dataset, num_replicas=world, rank=rank)
    return torch.utils.data.DataLoader(dataset, batch_size=args.batch_size, sampler=sampler,
                                       num_workers=args.num_workers, pin_memory=True, drop_last=True,
                                       collate_fn=ImageFolderTwoCrop.collate_fn, generator=torch.Generator())


def seed_epoch(loader, rng_seed, epoch, rank):
    """``moco_b200.augment.seed_epoch``, which both example drivers use; imported when called, as this module's
    other package imports are."""
    from moco_b200.augment import seed_epoch
    seed_epoch(loader, rng_seed, epoch, rank)


def main(argv=None):
    args = parse_args(argv)
    import torch
    import torch.distributed as dist
    from moco_b200 import checkpoint, encoders
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
    if args.steps is None:
        res = run_recipe(args, dev, rank, world)
        if world > 1:
            dist.barrier()
            dist.destroy_process_group()
        return res

    torch.manual_seed(0)
    ctor = getattr(encoders, args.arch)
    model = ctor(low_dim=128, width=args.model_width, mlp=args.mlp).to(dev).to(memory_format=torch.channels_last)
    model_ema = ctor(low_dim=128, width=args.model_width, mlp=args.mlp).to(dev).to(memory_format=torch.channels_last)
    moment_update(model, model_ema, 0)                                                    # train.py:133
    contrast = MemoryMoCo(128, args.nce_k, args.nce_t, persist_index=args.persist_index,
                          device_index=args.graph_tail).to(dev)                          # train.py:181
    opt = torch.optim.SGD(model.parameters(), lr=args.base_lr * args.batch_size * world / 256,
                          momentum=args.momentum, weight_decay=args.weight_decay)        # train.py:183-187
    if args.resume:
        ckpt = checkpoint.load(args.resume)                                              # train.py:157-166
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


def run_recipe(args, dev, rank, world):
    """train.py:175-293 on ``args.data_dir``/train.  Returns the last epoch's number, its mean loss and prob on this
    rank, its step count, and its wall time and the part of it spent waiting for batches, in seconds."""
    import time
    import torch
    from moco_b200 import checkpoint, encoders
    from moco_b200.augment import augment_two_crop, prefetch_pixels
    from moco_b200.linear_eval import get_scheduler
    from moco_b200.NCE import MemoryMoCo
    from moco_b200.train_step import MoCoStep
    from moco_b200.util import moment_update

    # fixed, deterministic cuDNN algorithms, as bench.py: a resumed run then computes what an uninterrupted one does
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    if rank == 0:
        print(f"--dataset {args.dataset} and --amp-opt-level {args.amp_opt_level} have no effect: the step always "
              "runs under bf16 autocast", flush=True)
    loader = make_recipe_loader(args, world, rank)
    n_iter = len(loader)
    if n_iter == 0:
        raise ValueError(f"{len(loader.dataset)} training images give no full batch of {args.batch_size} per rank")

    ckpt = checkpoint.load(args.resume) if args.resume else None
    if ckpt is not None and encoders.has_mlp_head(ckpt["model"]) != args.mlp:
        have = not args.mlp
        raise ValueError(f"--resume {args.resume}: its encoder has {'the' if have else 'no'} MLP head; resume it "
                         f"{'with' if have else 'without'} --mlp")
    torch.manual_seed(args.rng_seed)
    ctor = getattr(encoders, args.arch)
    model = ctor(low_dim=128, width=args.model_width, mlp=args.mlp).to(dev).to(memory_format=torch.channels_last)
    model_ema = ctor(low_dim=128, width=args.model_width, mlp=args.mlp).to(dev).to(memory_format=torch.channels_last)
    moment_update(model, model_ema, 0)                                                    # train.py:133
    contrast = MemoryMoCo(128, args.nce_k, args.nce_t, persist_index=args.persist_index,
                          device_index=args.graph_tail).to(dev)                          # train.py:181
    opt = torch.optim.SGD(model.parameters(), lr=args.batch_size * world / 256 * args.base_lr,
                          momentum=args.momentum, weight_decay=args.weight_decay)        # train.py:183-187
    scheduler = get_scheduler(opt, n_iter, args.epochs, args.lr_scheduler, args.warmup_epoch,
                              args.warmup_multiplier, args.lr_decay_epochs, args.lr_decay_rate)
    start_epoch = 1
    if ckpt is not None:
        start_epoch = checkpoint.restore(ckpt, model, model_ema, contrast, opt)
        scheduler.load_state_dict({"last_epoch": (start_epoch - 1) * n_iter})
        if rank == 0:
            print(f"resumed {args.resume}: epoch {start_epoch}, lr {opt.param_groups[0]['lr']:.6g}", flush=True)
    if world > 1:
        model = torch.nn.parallel.DistributedDataParallel(model, device_ids=[args.local_rank],
                                                          broadcast_buffers=False)     # train.py:198
    step = MoCoStep(model, model_ema, contrast, opt, alpha=args.alpha, channels_last=True,
                    fuse_normalize=args.fuse_normalize, graph_tail=args.graph_tail)
    if rank == 0:
        os.makedirs(args.output_dir, exist_ok=True)
        checkpoint.write_config(args, args.output_dir)                                  # train.py:305-309

    res = None
    for epoch in range(start_epoch, args.epochs + 1):
        seed_epoch(loader, args.rng_seed, epoch, rank)
        sums = torch.zeros(2, device=dev)                 # loss x batch, prob x batch: summed on the device
        seen, data_time, tic = 0, 0.0, time.perf_counter()
        end = tic
        for it, batch in enumerate(prefetch_pixels(loader, dev)):
            data_time += time.perf_counter() - end
            x1, x2 = torch.split(augment_two_crop(batch), [3, 3], dim=1)                 # train.py:250-254
            loss, prob = step(x1, x2, epoch)                                              # train.py:256-277
            scheduler.step()                                                              # train.py:275
            bsz = x1.shape[0]
            sums[0].add_(loss.detach(), alpha=bsz)
            sums[1].add_(prob.detach(), alpha=bsz)
            seen += bsz
            end = time.perf_counter()
            if rank == 0 and it % args.print_freq == 0:
                avg = (sums / seen).tolist()
                print(f"Train: [{epoch}][{it}/{n_iter}]  lr {opt.param_groups[0]['lr']:.4g}  "
                      f"loss {loss.item():.3f} ({avg[0]:.3f})  prob {prob.item():.3f} ({avg[1]:.3f})  "
                      f"T {(end - tic) / (it + 1):.3f}  DT {data_time / (it + 1):.3f}", flush=True)
        avg = (sums / seen).tolist()
        dt = time.perf_counter() - tic
        res = {"epoch": epoch, "loss": avg[0], "prob": avg[1], "steps": n_iter, "seconds": dt,
               "data_wait_seconds": data_time}
        if rank == 0:
            print(f"epoch {epoch}  loss {avg[0]:.4f}  prob {avg[1]:.4f}  time {dt:.2f} s  "
                  f"{seen * world / dt:.1f} img/s", flush=True)
            checkpoint.save(checkpoint.state(args, epoch, model, model_ema, contrast, opt, scheduler),
                            args.output_dir, args.save_freq)                             # train.py:227-228
    return res


def _cycle(loader):
    epoch = 0
    while True:
        if getattr(loader, "sampler", None) is not None and hasattr(loader.sampler, "set_epoch"):
            loader.sampler.set_epoch(epoch)                                              # train.py:213
        yield from loader
        epoch += 1


if __name__ == "__main__":
    main()
