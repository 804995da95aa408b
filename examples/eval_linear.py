"""Linear evaluation of a pretrained encoder -- the train / validate loop of bl0/moco's ``eval.py`` (eval.py:188-360)
on this package: a frozen ResNet-50 (``MoCoResNet.freeze()``, whose BatchNorms run on the eval kernels) feeds the
features of ``--layer`` to the reference's linear classifier (``moco_b200.linear_eval``), trained with SGD (lr 30,
momentum 0.9, no weight decay) and cross-entropy; top-1 / top-5 accuracy.

With ``--data-dir`` (``train/`` and ``val/`` image folders under it, as eval.py:119-120) it runs eval.py's recipe on
real images: ``n_label`` is the folder's class count; the workers only decode (``moco_b200.augment.ImageFolderEval``)
and the GPU applies the train crops (``augment_crops``, ``--aug``, ``--crop``) and the validation Resize(256) ->
CenterCrop(224) (``resize_center_crops``); the learning rate follows eval.py's warm-up + cosine / step schedule per
iteration (``moco_b200.linear_eval.get_scheduler``); every epoch trains, then validates over the whole validation set
split across ranks without padding, and rank 0 prints ``* Acc@1 ... Acc@5 ... (n = ...)``.  Without ``--data-dir``
synthetic images and labels stand in for the dataset (``--steps`` / ``--val-steps``, constant learning rate).

``--pretrained`` takes a checkpoint written by ``examples/train_moco.py --save`` or by the reference's ``train.py``:
its ``model`` entry in either key naming, with or without the ``module.`` prefix.  Launch as train_moco.py
(``--local_rank`` / ``--local-rank`` / ``$LOCAL_RANK``); with more than one process the classifier is wrapped in
DistributedDataParallel as eval.py:211 does.

    python examples/eval_linear.py --pretrained ckpt.pth --steps 20
    torchrun --nproc_per_node 8 examples/eval_linear.py --pretrained ckpt.pth --data-dir /data/imagenet
"""
import argparse
import os


def parse_args(argv=None):
    ap = argparse.ArgumentParser("moco_b200 linear evaluation")
    ap.add_argument("--local_rank", "--local-rank", dest="local_rank", type=int,
                    default=int(os.environ.get("LOCAL_RANK", 0)), help="GPU of this process (default: $LOCAL_RANK)")
    ap.add_argument("--pretrained", "--pretrained-model", dest="pretrained", default="",
                    help="pretrained checkpoint (either key naming); random weights when empty")
    ap.add_argument("--model-width", type=int, default=1)
    ap.add_argument("--layer", type=int, default=6, choices=[2, 3, 4, 5, 6],
                    help="which layer to evaluate (2..6; the reference's classifier sizes layer 1 for 128 channels, "
                         "where both models give 64)")
    ap.add_argument("--num-classes", type=int, default=1000)
    ap.add_argument("--total-batch-size", type=int, default=256, help="over all GPUs (eval.py: --total-batch-size)")
    ap.add_argument("--learning-rate", type=float, default=30.0)
    ap.add_argument("--momentum", type=float, default=0.9)
    ap.add_argument("--weight-decay", type=float, default=0.0)
    ap.add_argument("--steps", type=int, default=20, help="training steps")
    ap.add_argument("--val-steps", type=int, default=2)
    ap.add_argument("--print-freq", type=int, default=10)
    # real data (eval.py's flags and defaults); without --data-dir the synthetic loop above runs
    ap.add_argument("--data-dir", default="", help="root with train/ and val/ image folders (default: synthetic data)")
    ap.add_argument("--aug", default="NULL", choices=["NULL", "CJ"], help="train augmentation (eval.py: --aug)")
    ap.add_argument("--crop", type=float, default=0.08, help="RandomResizedCrop's minimum scale")
    ap.add_argument("--num-workers", type=int, default=4)
    ap.add_argument("--epochs", type=int, default=100)
    ap.add_argument("--lr-scheduler", default="cosine", choices=["step", "cosine"])
    ap.add_argument("--warmup-epoch", type=int, default=5)
    ap.add_argument("--warmup-multiplier", type=int, default=100)
    ap.add_argument("--lr-decay-epochs", type=int, default=[30, 60, 90], nargs="+")
    ap.add_argument("--lr-decay-rate", type=float, default=0.1)
    return ap.parse_args(argv)


def accuracy(output, target, topk=(1, 5)):
    """Top-k accuracy in percent (moco/util.py:accuracy)."""
    maxk = max(topk)
    _, pred = output.topk(maxk, 1, True, True)
    correct = pred.t().eq(target.view(1, -1).expand_as(pred.t()))
    return [correct[:k].reshape(-1).float().sum() * (100.0 / target.size(0)) for k in topk]


def main(argv=None):
    args = parse_args(argv)
    import torch
    import torch.distributed as dist
    from moco_b200.encoders import from_reference_state_dict, resnet50
    from moco_b200.linear_eval import LinearClassifierResNet

    world = int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(args.local_rank)
    dev = torch.device("cuda", args.local_rank)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
    rank = dist.get_rank() if world > 1 else 0
    torch.manual_seed(0)

    model = resnet50(width=args.model_width).to(dev).to(memory_format=torch.channels_last)
    if args.pretrained:                                                                  # eval.py:149-153
        ckpt = torch.load(args.pretrained, map_location="cpu")
        model.load_state_dict(from_reference_state_dict(ckpt["model"]))
        if rank == 0:
            print(f"loaded {args.pretrained} (epoch {ckpt.get('epoch', '?')})", flush=True)
    model.freeze()
    if args.data_dir:
        res = run_data(args, model, dev, rank, world)
        if world > 1:
            dist.barrier()
            dist.destroy_process_group()
        return res
    classifier = LinearClassifierResNet(args.layer, args.num_classes, "avg", args.model_width).to(dev)
    criterion = torch.nn.CrossEntropyLoss()
    optimizer = torch.optim.SGD(classifier.parameters(), lr=args.learning_rate, momentum=args.momentum,
                                weight_decay=args.weight_decay)
    if world > 1:
        classifier = torch.nn.parallel.DistributedDataParallel(classifier, device_ids=[args.local_rank],
                                                               broadcast_buffers=False)

    batch = args.total_batch_size // world
    gen = torch.Generator(device=dev).manual_seed(1234 + rank)

    def features(x):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            return model(x, args.layer).float()

    classifier.train()                                                                    # eval.py:254-311
    for it in range(args.steps):
        x = torch.randn(batch, 3, 224, 224, device=dev, generator=gen)
        y = torch.randint(0, args.num_classes, (batch,), device=dev, generator=gen)
        output = classifier(features(x))
        loss = criterion(output, y)
        acc1, acc5 = accuracy(output, y)
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
        if rank == 0 and (it % args.print_freq == 0 or it == args.steps - 1):
            print(f"step {it:4d}  loss {loss.item():.4f}  acc@1 {acc1.item():.3f}  acc@5 {acc5.item():.3f}", flush=True)

    classifier.eval()                                                                     # eval.py:314-360
    with torch.no_grad():
        tot = torch.zeros(3, device=dev)
        for _ in range(args.val_steps):
            x = torch.randn(batch, 3, 224, 224, device=dev, generator=gen)
            y = torch.randint(0, args.num_classes, (batch,), device=dev, generator=gen)
            output = classifier(features(x))
            acc1, acc5 = accuracy(output, y)
            tot += torch.stack([criterion(output, y), acc1, acc5]) / max(args.val_steps, 1)
        if world > 1:
            dist.all_reduce(tot)
            tot /= world
    if rank == 0:
        print(f"val  loss {tot[0].item():.4f}  acc@1 {tot[1].item():.3f}  acc@5 {tot[2].item():.3f}", flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def run_data(args, model, dev, rank, world):
    """eval.py:188-360 on the image folders under args.data_dir."""
    import torch
    from torch.utils.data import DataLoader, DistributedSampler
    from moco_b200 import augment as A
    from moco_b200.linear_eval import LinearClassifierResNet, ShardSampler, finish_validation, get_scheduler, val_totals

    train_ds = A.ImageFolderEval(os.path.join(args.data_dir, "train"), train=True, scale=(args.crop, 1.0),
                                 aug=args.aug)
    val_ds = A.ImageFolderEval(os.path.join(args.data_dir, "val"), train=False)
    batch = args.total_batch_size // world
    train_sampler = DistributedSampler(train_ds, num_replicas=world, rank=rank)
    train_loader = DataLoader(train_ds, batch_size=batch, sampler=train_sampler, num_workers=args.num_workers,
                              pin_memory=True, drop_last=True, collate_fn=train_ds.collate_fn)
    val_loader = DataLoader(val_ds, batch_size=batch, sampler=ShardSampler(len(val_ds), rank, world),
                            num_workers=args.num_workers, pin_memory=True, drop_last=False,
                            collate_fn=val_ds.collate_fn)
    if len(train_loader) == 0:
        raise ValueError(f"{len(train_ds)} training images give no full batch of {batch} per rank")
    n_label = len(train_ds.classes)
    if rank == 0:
        print(f"train: {len(train_ds)} images, val: {len(val_ds)} images, {n_label} classes", flush=True)

    classifier = LinearClassifierResNet(args.layer, n_label, "avg", args.model_width).to(dev)
    criterion = torch.nn.CrossEntropyLoss()
    optimizer = torch.optim.SGD(classifier.parameters(), lr=args.learning_rate, momentum=args.momentum,
                                weight_decay=args.weight_decay)
    scheduler = get_scheduler(optimizer, len(train_loader), args.epochs, args.lr_scheduler, args.warmup_epoch,
                              args.warmup_multiplier, args.lr_decay_epochs, args.lr_decay_rate)
    if world > 1:
        classifier = torch.nn.parallel.DistributedDataParallel(classifier, device_ids=[args.local_rank],
                                                               broadcast_buffers=False)

    def features(x):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            return model(x, args.layer).float()

    for epoch in range(1, args.epochs + 1):
        train_sampler.set_epoch(epoch)
        classifier.train()
        for it, b in enumerate(train_loader):                                             # eval.py:254-311
            x = A.augment_crops(b, dtype=torch.bfloat16, device=dev)
            y = b[2].to(dev, non_blocking=True)
            output = classifier(features(x))
            loss = criterion(output, y)
            optimizer.zero_grad()
            loss.backward()
            optimizer.step()
            scheduler.step()
            if rank == 0 and it % args.print_freq == 0:
                print(f"epoch {epoch} [{it}/{len(train_loader)}]  lr {optimizer.param_groups[0]['lr']:.4g}  "
                      f"loss {loss.item():.4f}", flush=True)

        classifier.eval()                                                                 # eval.py:314-360
        totals = torch.zeros(4, dtype=torch.float64, device=dev)
        with torch.no_grad():
            for b in val_loader:
                x = A.resize_center_crops(b, dtype=torch.bfloat16, device=dev)
                y = b[2].to(dev, non_blocking=True)
                output = classifier(features(x))
                totals += val_totals(output, y, criterion(output, y))
        res = finish_validation(totals, len(val_ds))
        if rank == 0:
            print(f" * Acc@1 {res['acc'][0]:.3f} Acc@5 {res['acc'][1]:.3f} (n = {res['n']})  loss {res['loss']:.4f}",
                  flush=True)
    return res


if __name__ == "__main__":
    main()
