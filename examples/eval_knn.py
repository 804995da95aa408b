"""Weighted kNN evaluation of a pretrained encoder: is this checkpoint any good yet, without training a classifier.

The frozen encoder (``MoCoResNet.freeze()``) turns the ``train/`` images under ``--data-dir`` into an L2-normalised
feature bank (``moco_b200.knn.build_bank``), then each ``val/`` image is classified by the weighted vote of its
``--knn-k`` nearest bank rows, weights exp(s / ``--knn-t``) (``knn_evaluate`` on ``moco_knn``, which never stores
the similarity matrix).  Both splits take the validation transform, Resize(256) -> CenterCrop(224) -> Normalize
(``augment.ImageFolderEval(train=False)`` decoded by the workers, ``resize_center_crops`` on the GPU): the train images
are not augmented.  ``--layer 7`` is the fc output the contrast head trains (128-d), ``--layer 6`` the pooled 2048-d
features.  Rank 0 prints ``* kNN Acc@1 ... Acc@5 ... (n = ...)``, over exactly the validation set's images.

``--pretrained-model`` takes a checkpoint of either project (``examples/train_moco.py`` or the reference's
``train.py``): its ``model`` entry in either key naming, with or without the ``module.`` prefix.  Launch as the
other examples (``--local_rank`` / ``--local-rank`` / ``$LOCAL_RANK``); with more than one process each extracts its
share of the train set and one all-gather gives every rank the same bank, whatever the world size.

    python examples/eval_knn.py --data-dir /data/imagenet --pretrained-model ./output/current.pth
    torchrun --nproc_per_node 8 examples/eval_knn.py --data-dir /data/imagenet --pretrained-model ckpt.pth
"""
import argparse
import os


def parse_args(argv=None):
    ap = argparse.ArgumentParser("moco_b200 kNN evaluation")
    ap.add_argument("--local_rank", "--local-rank", dest="local_rank", type=int,
                    default=int(os.environ.get("LOCAL_RANK", 0)), help="GPU of this process (default: $LOCAL_RANK)")
    ap.add_argument("--data-dir", required=True, help="root with train/ and val/ image folders")
    ap.add_argument("--pretrained", "--pretrained-model", dest="pretrained", required=True,
                    help="pre-training checkpoint of either project, either key naming")
    ap.add_argument("--model-width", type=int, default=1)
    ap.add_argument("--layer", type=int, default=7, choices=[6, 7],
                    help="7: the 128-d fc output (default); 6: the pooled features, L2-normalised")
    ap.add_argument("--knn-k", type=int, default=200,
                    help="neighbours per query, at most 1024 (default 200, lemniscate.pytorch's kNN setting)")
    ap.add_argument("--knn-t", type=float, default=0.07,
                    help="temperature of the weights exp(s / T) (default 0.07: lemniscate.pytorch's kNN setting and "
                         "the reference's --nce-t default)")
    ap.add_argument("--total-batch-size", type=int, default=256, help="over all GPUs")
    ap.add_argument("--num-workers", type=int, default=4)
    args = ap.parse_args(argv)
    if not 1 <= args.knn_k <= 1024:
        ap.error(f"--knn-k must be in [1, 1024] (got {args.knn_k})")
    if not args.knn_t > 0:
        ap.error(f"--knn-t must be > 0 (got {args.knn_t})")
    if args.total_batch_size < 1:
        ap.error("--total-batch-size must be at least 1")
    return args


def main(argv=None):
    """Returns {"n", "acc": [top-1, top-5], "bank": (Nb, C)}."""
    args = parse_args(argv)
    import time
    import torch
    import torch.distributed as dist
    from torch.utils.data import DataLoader
    from moco_b200 import augment as A
    from moco_b200 import checkpoint
    from moco_b200.encoders import encoder_from_state_dict
    from moco_b200.knn import build_bank, knn_evaluate
    from moco_b200.linear_eval import ShardSampler

    world = int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(args.local_rank)
    dev = torch.device("cuda", args.local_rank)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
    rank = dist.get_rank() if world > 1 else 0
    t0 = time.perf_counter()

    ckpt = checkpoint.load(args.pretrained)
    model = encoder_from_state_dict(ckpt["model"], width=args.model_width)   # with the MLP head an --mlp run trained
    model = model.to(dev).to(memory_format=torch.channels_last)
    model.freeze()
    if rank == 0:
        print(f"loaded {args.pretrained} (epoch {ckpt.get('epoch', '?')})", flush=True)

    batch = max(args.total_batch_size // world, 1)

    def loader(split):
        ds = A.ImageFolderEval(os.path.join(args.data_dir, split), train=False)
        return DataLoader(ds, batch_size=batch, sampler=ShardSampler(len(ds), rank, world),
                          num_workers=args.num_workers, pin_memory=True, drop_last=False, collate_fn=ds.collate_fn)

    train_loader, val_loader = loader("train"), loader("val")
    n_classes = len(train_loader.dataset.classes)
    bank, labels = build_bank(model, train_loader, args.layer, dev)
    if rank == 0:
        print(f"bank: {bank.shape[0]} x {bank.shape[1]} (layer {args.layer}), {n_classes} classes, "
              f"val: {len(val_loader.dataset)} images", flush=True)
    res = knn_evaluate(model, bank, labels, val_loader, args.knn_k, args.knn_t, args.layer, n_classes, dev)
    if rank == 0:
        print(f" * kNN Acc@1 {res['acc'][0]:.3f} Acc@5 {res['acc'][1]:.3f} (n = {res['n']})  k {args.knn_k}  "
              f"T {args.knn_t}  {time.perf_counter() - t0:.1f} s", flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return {"n": res["n"], "acc": res["acc"], "bank": tuple(bank.shape)}


if __name__ == "__main__":
    main()
