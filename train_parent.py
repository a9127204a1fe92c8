#!/usr/bin/env python
"""Parent-network training entry point - same role and defaults as the reference's train_parent.py
(240 epochs, deep-supervision loss, SGD lr 1e-8), plus the data-parallel path the reference lacks:

    python train_parent.py --synthetic --epochs 1 --iters-per-epoch 20                      # 1 GPU
    torchrun --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 train_parent.py --synthetic ...   # 8 GPUs

Each rank holds `--batch` frames per micro-batch; gradients are averaged over ranks once per optimizer
step (osvos_pytorch_b200/parallel.py).  R ranks x batch b reproduces the reference run with
trainBatch = b, nAveGrad = R (--n-ave-grad then counts additional LOCAL accumulation)."""
import argparse
import os
import timeit

import torch
import torch.distributed as dist

import networks.vgg_osvos as vo
from mypath import Path
from osvos_pytorch_b200 import evaluation, ops, parallel, training


class _Mapped:
    """A re-iterable view of a DataLoader with ``fn`` applied to every batch (keeps ``len``)."""

    def __init__(self, loader, fn):
        self.loader, self.fn = loader, fn

    def __len__(self):
        return len(self.loader)

    def __iter__(self):
        return (self.fn(b) for b in self.loader)


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=240)
    ap.add_argument("--resume-epoch", type=int, default=0)
    ap.add_argument("--batch", type=int, default=1, help="frames per rank per micro-batch (reference trainBatch)")
    ap.add_argument("--n-ave-grad", type=int, default=None,
                    help="local micro-batches per optimizer step (default: 10 / world size, at least 1)")
    ap.add_argument("--snapshot", type=int, default=40)
    ap.add_argument("--test-interval", type=int, default=5)
    ap.add_argument("--lr", type=float, default=1e-8)
    ap.add_argument("--wd", type=float, default=0.0002)
    ap.add_argument("--pretrained", type=int, default=2, help="2 = Caffe VGG (.mat), 1 = torchvision VGG, 0 = none")
    ap.add_argument("--precision", default="exact", choices=["exact", "fast"])
    ap.add_argument("--synthetic", action="store_true")
    ap.add_argument("--iters-per-epoch", type=int, default=2079, help="synthetic mode: micro-batches per epoch (global)")
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=854)
    ap.add_argument("--model-name", default="parent")
    ap.add_argument("--loader", default="reference", choices=["reference", "native"],
                    help="real data: the reference's dataloaders package (reference), or osvos_pytorch_b200.davis "
                         "(native: workers only decode; ingest and augmentation run on the device)")
    ap.add_argument("--workers", type=int, default=2, help="DataLoader decode workers per rank")
    ap.add_argument("--val-measures", action="store_true",
                    help="also score every validation frame on the device (DAVIS-2016 J and F, mean over sequences); "
                         "needs --loader native")
    a = ap.parse_args(argv)
    if a.val_measures and (a.synthetic or a.loader != "native"):
        ap.error("--val-measures scores against the DAVIS annotations read by --loader native; it cannot be combined "
                 "with " + ("--synthetic" if a.synthetic else "--loader reference"))
    return a


def _val_scores(per_seq):
    """{sequence: SequenceScores} -> the dataset means over sequences of the J and F statistics."""
    import numpy as np
    stats = [sc.result()["statistics"] for sc in per_seq.values()]
    return {m: {k: float(np.mean([st[m][k] for st in stats])) if stats else float("nan") for k in "MOD"}
            for m in ("J", "F")}


def main(argv=None):
    a = parse(argv)
    rank, world, local = parallel.init_distributed()
    device = torch.device("cuda", local)
    torch.cuda.set_device(device)
    n_ave = a.n_ave_grad if a.n_ave_grad is not None else max(1, 10 // world)
    save_dir = Path.save_root_dir()
    os.makedirs(save_dir, exist_ok=True)

    if a.resume_epoch == 0:
        net = vo.OSVOS(pretrained=0 if a.synthetic else a.pretrained, precision=a.precision, verbose=rank == 0)
        if a.synthetic:
            vo.he_init_(net, seed=0)
    else:
        net = vo.OSVOS(pretrained=0, precision=a.precision, verbose=rank == 0)
        ckpt = os.path.join(save_dir, f"{a.model_name}_epoch-{a.resume_epoch - 1}.pth")
        net.load_state_dict(torch.load(ckpt, map_location="cpu"))
    net.to(device)
    parallel.broadcast_parameters(net, src=0)        # replicas must be ONE model (the reference's init is unseeded)
    opt = training.make_optimizer(net, "parent", a.lr, a.wd, fused=True)
    bucket = parallel.GradientBucket(parallel.trainable_parameters(net), device)

    if a.synthetic:
        def epoch_batches(epoch):
            # the same number of micro-batches on every rank (a multiple of n_ave): every rank joins every allreduce
            per = parallel.steps_per_rank(a.iters_per_epoch, world, n_ave)
            if per == 0:
                raise ValueError(f"--iters-per-epoch {a.iters_per_epoch} gives no complete optimizer step on {world} ranks with "
                                 f"nAveGrad {n_ave} (need >= {world * n_ave})")
            for i in range(rank * per, (rank + 1) * per):
                yield training.synthetic_batch(a.batch, a.height, a.width, 7919 * epoch + i, device)
        val_batches = None
    elif a.loader == "native":
        import random
        from torch.utils.data import DataLoader
        from torch.utils.data.distributed import DistributedSampler
        from osvos_pytorch_b200 import davis
        db_train = davis.DAVIS2016Frames(train=True, db_root_dir=Path.db_root_dir())
        sampler = DistributedSampler(db_train, world, rank, shuffle=True, drop_last=True) if world > 1 else None
        loader = DataLoader(db_train, batch_size=a.batch, shuffle=sampler is None, sampler=sampler, num_workers=a.workers,
                            drop_last=world > 1, collate_fn=davis.collate,
                            persistent_workers=a.workers > 0)
        db_test = davis.DAVIS2016Frames(train=False, db_root_dir=Path.db_root_dir())
        # no pin_memory=True: to_device pins in this thread (davis.pinned says why)
        val_loader = DataLoader(db_test, batch_size=1, shuffle=False, num_workers=a.workers, collate_fn=davis.collate)
        if a.val_measures:
            def val_item(b):                         # davis.to_device without augmentation, keeping the mask bytes
                with torch.cuda.device(device):
                    img, gt, stats = davis.upload(b, device)
                    return {"image": ops.image_from_bgr8(img), "gt": ops.label_from_u8(gt, stats), "gt_u8": gt,
                            "fname": b["fname"]}
            val_batches = _Mapped(val_loader, val_item)
        else:
            val_batches = _Mapped(val_loader, lambda b: davis.to_device(b, device))

        def epoch_batches(epoch):
            if sampler is not None:
                sampler.set_epoch(epoch)
            for b in loader:      # flip / rotation / scale drawn from Python's random, as the reference's transforms do
                yield davis.to_device(b, device, augment=random)
    else:
        from dataloaders import davis_2016 as db
        from dataloaders import custom_transforms as tr
        from torch.utils.data import DataLoader
        from torch.utils.data.distributed import DistributedSampler
        from torchvision import transforms
        aug = transforms.Compose([tr.RandomHorizontalFlip(), tr.ScaleNRotate(rots=(-30, 30), scales=(.75, 1.25)),
                                  tr.ToTensor()])
        db_train = db.DAVIS2016(train=True, inputRes=None, db_root_dir=Path.db_root_dir(), transform=aug)
        sampler = DistributedSampler(db_train, world, rank, shuffle=True, drop_last=True) if world > 1 else None
        loader = DataLoader(db_train, batch_size=a.batch, shuffle=sampler is None, sampler=sampler, num_workers=2,
                            drop_last=world > 1)
        db_test = db.DAVIS2016(train=False, db_root_dir=Path.db_root_dir(), transform=tr.ToTensor())
        val_batches = DataLoader(db_test, batch_size=1, shuffle=False, num_workers=2)

        def epoch_batches(epoch):
            if sampler is not None:
                sampler.set_epoch(epoch)
            for s in loader:
                yield {"image": s["image"].to(device, non_blocking=True), "gt": s["gt"].to(device, non_blocking=True)}

    if rank == 0:
        print(f"Training Network on {world} GPU(s): batch/rank {a.batch}, local nAveGrad {n_ave}, "
              f"gradient allreduce payload {bucket.numel * 4 / 1e6:.1f} MB per optimizer step")
    loop_state = {}                                  # accumulation counter, carried across epochs as in the reference
    for epoch in range(a.resume_epoch, a.epochs):
        t0 = timeit.default_timer()
        losses = training.parent_epoch(net, opt, bucket, epoch_batches(epoch), epoch, a.epochs, n_ave, state=loop_state)
        torch.cuda.synchronize()
        if rank == 0:
            print(f"[Epoch: {epoch}] " + " ".join(f"Loss {k}: {v:.4f}" for k, v in enumerate(losses.tolist()))
                  + f"  Execution time: {timeit.default_timer() - t0:.2f}")
            if epoch % a.snapshot == a.snapshot - 1 and epoch != 0:
                torch.save(net.state_dict(), os.path.join(save_dir, f"{a.model_name}_epoch-{epoch}.pth"))
        if val_batches is not None and rank == 0 and epoch % a.test_interval == a.test_interval - 1:
            net.eval()
            tot = torch.zeros(5, device=device)
            per_seq = {}
            with torch.no_grad():
                for s in val_batches:
                    outs = net.forward(s["image"].to(device))
                    tot += torch.stack([training.class_balanced_cross_entropy_loss(o, s["gt"].to(device),
                                                                                   size_average=False) for o in outs])
                    if a.val_measures:
                        counts = ops.davis_measures(outs[-1], s["gt_u8"])
                        for i, fname in enumerate(s["fname"]):
                            per_seq.setdefault(fname.split("/")[0], evaluation.SequenceScores()).add(counts[i:i + 1])
            print("***Testing *** " + " ".join(f"Loss {k}: {v:.4f}" for k, v in enumerate((tot / len(val_batches)).tolist())))
            if a.val_measures:
                sc = _val_scores(per_seq)
                print("***Testing *** " + "  ".join(f"{m} M/O/D: {sc[m]['M']:.4f} / {sc[m]['O']:.4f} / {sc[m]['D']:.4f}"
                                                    for m in ("J", "F")) + f"  ({len(per_seq)} sequences)")
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
