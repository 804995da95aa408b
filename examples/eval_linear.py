"""Linear evaluation of a pretrained encoder -- the train / validate loop of bl0/moco's ``eval.py`` (eval.py:188-360)
on this package: a frozen ResNet-50 (``MoCoResNet.freeze()``, whose BatchNorms run on the eval kernels) feeds the
features of ``--layer`` to the reference's linear classifier (``moco_b200.linear_eval``), trained with SGD (lr 30,
momentum 0.9, no weight decay) and cross-entropy; top-1 / top-5 accuracy.  Synthetic images and labels stand in for
the dataset (the reference's dataset, augmentation and LR schedule are out of scope).

``--pretrained`` takes a checkpoint written by ``examples/train_moco.py --save`` or by the reference's ``train.py``:
its ``model`` entry in either key naming, with or without the ``module.`` prefix.  Launch as train_moco.py
(``--local_rank`` / ``--local-rank`` / ``$LOCAL_RANK``); with more than one process the classifier is wrapped in
DistributedDataParallel as eval.py:211 does.

    python examples/eval_linear.py --pretrained ckpt.pth --steps 20
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


if __name__ == "__main__":
    main()
