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
    ap.add_argument("--upsampling-lr", type=float, default=0.0,
                    help="lr of the side-output deconvolutions (upscale / upscale_); 0 keeps them fixed as the reference "
                         "does, a nonzero value trains them (the net learns its upsampling)")
    ap.add_argument("--deterministic", action="store_true",
                    help="torch.use_deterministic_algorithms(True) before anything is built: the package's kernels "
                         "reduce in a fixed order, so two runs on the same device give bit-identical results")
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
    ap.add_argument("--cache", default="none", choices=["none", "device"],
                    help="device: decode the train split once and keep its bytes on every GPU (about 3.4 GB per rank, "
                         "plus 2.3 GB of val frames on rank 0), then augment each batch from there instead of "
                         "decoding every frame in every epoch; needs --loader native")
    ap.add_argument("--decode", default="host", choices=["host", "device"],
                    help="--loader native: decode the JPEG frames with cv2.imread in the workers (host), or parse them "
                         "there and decode them on the GPU, bit-identically (device; files outside the decoder's subset "
                         "still go through cv2.imread)")
    ap.add_argument("--input-res", type=int, nargs=2, default=None, metavar=("H", "W"),
                    help="the reference's inputRes: resize every frame (bilinear) and annotation (nearest) to H x W on "
                         "the device, before augmentation and validation, as scipy 1.0's imresize does. Needs --loader "
                         "native (--synthetic has --height / --width)")
    ap.add_argument("--output-res", default="network", choices=["network", "stored"],
                    help="with --input-res and --val-measures: score J and F at the network resolution against the "
                         "nearest-resized annotations (network), or upsample the fused logits to each frame's stored "
                         "size on the device, as scipy 1.0's imresize(mode='F') does, and score them against the "
                         "original annotations (stored). The validation loss stays at the network resolution")
    ap.add_argument("--davis", default="2016", choices=["2016", "2017"],
                    help="2017: train on ImageSets/2017/train.txt with every object as foreground and void (255) pixels "
                         "left out of the loss, validate on val.txt (--val-measures: J and F of the union of the "
                         "objects, void ignored); needs --loader native")
    a = ap.parse_args(argv)
    if a.davis == "2017":
        if a.synthetic or a.loader != "native":
            ap.error("--davis 2017 reads DAVIS-2017 with --loader native; it cannot be combined with "
                     + ("--synthetic" if a.synthetic else "--loader reference"))
        if a.upsampling_lr != 0.0:
            ap.error("--davis 2017 trains with void labels, which the learned-upsampling tail does not support; it "
                     "cannot be combined with a nonzero --upsampling-lr")
    if a.val_measures and (a.synthetic or a.loader != "native"):
        ap.error("--val-measures scores against the DAVIS annotations read by --loader native; it cannot be combined "
                 "with " + ("--synthetic" if a.synthetic else "--loader reference"))
    if a.cache == "device" and (a.synthetic or a.loader != "native"):
        ap.error("--cache device keeps the frames decoded by --loader native on the device; it cannot be combined "
                 "with " + ("--synthetic" if a.synthetic else "--loader reference"))
    if a.input_res is not None and (a.synthetic or a.loader != "native"):
        ap.error("--input-res resizes the frames read by --loader native; it cannot be combined with "
                 + ("--synthetic (use --height / --width)" if a.synthetic else "--loader reference"))
    if a.decode == "device" and (a.synthetic or a.loader != "native"):
        ap.error("--decode device decodes the frames read by --loader native; it cannot be combined with "
                 + ("--synthetic" if a.synthetic else "--loader reference"))
    return a


def main(argv=None):
    a = parse(argv)
    if a.deterministic:
        torch.use_deterministic_algorithms(True)
    rank, world, local = parallel.init_distributed()
    device = torch.device("cuda", local)
    torch.cuda.set_device(device)
    n_ave = a.n_ave_grad if a.n_ave_grad is not None else max(1, 10 // world)
    save_dir = Path.save_root_dir()
    os.makedirs(save_dir, exist_ok=True)

    if a.resume_epoch == 0:
        net = vo.OSVOS(pretrained=0 if a.synthetic else a.pretrained, precision=a.precision, verbose=rank == 0,
                       learn_upsampling=a.upsampling_lr != 0.0)
        if a.synthetic:
            vo.he_init_(net, seed=0)
    else:
        net = vo.OSVOS(pretrained=0, precision=a.precision, verbose=rank == 0, learn_upsampling=a.upsampling_lr != 0.0)
        ckpt = os.path.join(save_dir, f"{a.model_name}_epoch-{a.resume_epoch - 1}.pth")
        net.load_state_dict(torch.load(ckpt, map_location="cpu"))
    net.to(device)
    parallel.broadcast_parameters(net, src=0)        # replicas must be ONE model (the reference's init is unseeded)
    opt = training.make_optimizer(net, "parent", a.lr, a.wd, fused=True, upsampling_lr=a.upsampling_lr)
    bucket = parallel.GradientBucket(parallel.trainable_parameters(net), device)

    stored = False                                   # J and F at the stored size (--input-res --output-res stored)
    void = a.davis == "2017"                         # DAVIS-2017: labels from object ids, void left out of the loss

    def gt_label(gt, stats):
        return ops.labels_from_ids(gt, "all") if void else ops.label_from_u8(gt, stats)

    def measures(logits, gt_u8):
        if not void:
            return ops.davis_measures(logits, gt_u8)
        # the union of the objects: the fused map > 0 against every object id (void, 255, kept and ignored)
        union = torch.where(gt_u8 == 255, gt_u8, (gt_u8 != 0).to(torch.uint8))
        return ops.davis_measures_objects((logits > 0).to(torch.uint8), union, 1)
    jpeg_status = None                               # --decode device, streaming: the decoder's status words, summed
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
        if void:                                     # object ids: labels 1 (any object), 0, -1 (void)
            db_train = davis.DAVIS2017Frames("train", db_root_dir=Path.db_root_dir(), decode=a.decode)
            db_test = davis.DAVIS2017Frames("val", db_root_dir=Path.db_root_dir(), decode=a.decode)
        else:
            db_train = davis.DAVIS2016Frames(train=True, db_root_dir=Path.db_root_dir(), decode=a.decode)
            db_test = davis.DAVIS2016Frames(train=False, db_root_dir=Path.db_root_dir(), decode=a.decode)
        ids = "all" if void else False
        sampler = DistributedSampler(db_train, world, rank, shuffle=True, drop_last=True) if world > 1 else None
        res = None if a.input_res is None else tuple(a.input_res)
        stored = res is not None and a.val_measures and a.output_res == "stored"
        if res is not None and rank == 0:
            print(f"Frames resized to {res[0]}x{res[1]} (inputRes)"
                  + ("; validation J and F scored at the stored size (fused logits upsampled) against the original "
                     "annotations" if stored else
                     "; validation scored against the nearest-resized annotations" if a.val_measures else ""))
        if a.cache == "device":
            # The stores replace the decoding loaders.  Index loaders with the streaming loaders' batching and sampling
            # and no workers draw from the global RNG as 0-worker streaming loaders do (one base seed per pass, then
            # the sampler's own draw), so a seeded run sees the same batches and the same augmentation draws.
            train_store = davis.DeviceFrames(db_train, device, workers=a.workers,
                                             group=dist.group.WORLD if world > 1 else None, input_res=res)
            loader = DataLoader(range(len(db_train)), batch_size=a.batch, shuffle=sampler is None, sampler=sampler,
                                num_workers=0, drop_last=world > 1)
            val_batches = None
            if rank == 0:                            # only rank 0 validates
                val_store = davis.DeviceFrames(db_test, device, workers=a.workers, input_res=res, keep_stored_gt=stored)
                val_batches = _Mapped(DataLoader(range(len(db_test)), batch_size=1, shuffle=False, num_workers=0),
                                      lambda b: val_store.ingest(int(b[0])))
                for name, st in (("train", train_store), ("val", val_store)):
                    print(f"Device frame store ({name}): {len(st)} frames, {st.nbytes / 1e9:.2f} GB, built in "
                          f"{st.build_s:.1f} s" + (f"; {st.fallback_frames} frames decoded by cv2.imread, "
                                                   f"{st.redecoded_frames} re-decoded after a decoder status"
                                                   if a.decode == "device" else ""))

            def epoch_batches(epoch):
                if sampler is not None:
                    sampler.set_epoch(epoch)
                yield from train_store.batches(loader, rng=random)
        else:
            if a.decode == "device":
                jpeg_status = torch.zeros(1, dtype=torch.int32, device=device)
            loader = DataLoader(db_train, batch_size=a.batch, shuffle=sampler is None, sampler=sampler,
                                num_workers=a.workers, drop_last=world > 1, collate_fn=davis.collate,
                                persistent_workers=a.workers > 0)
            # no pin_memory=True: to_device pins in this thread (davis.pinned says why)
            val_loader = DataLoader(db_test, batch_size=1, shuffle=False, num_workers=a.workers,
                                    collate_fn=davis.collate)
            if a.val_measures:
                def val_item(b):                     # davis.to_device without augmentation, keeping the mask bytes
                    with torch.cuda.device(device):
                        if not stored:
                            img, gt, stats = davis.upload(b, device, input_res=res, jpeg_status=jpeg_status)
                            return {"image": ops.image_from_bgr8(img), "gt": gt_label(gt, stats), "gt_u8": gt,
                                    "fname": b["fname"]}
                        # davis.upload, keeping the collated mask's view at the stored size
                        img0, gt0, _ = davis.device_views(b, device, jpeg_status)
                        img, gt = davis.resize_pair(img0, gt0, res)
                        stats = ops.label_stats_u8(gt)
                        return {"image": ops.image_from_bgr8(img), "gt": gt_label(gt, stats), "gt_u8": gt,
                                "gt_u8_stored": gt0, "fname": b["fname"]}
                val_batches = _Mapped(val_loader, val_item)
            else:
                val_batches = _Mapped(val_loader, lambda b: davis.to_device(b, device, input_res=res,
                                                                            jpeg_status=jpeg_status, ids=ids))

            def epoch_batches(epoch):
                if sampler is not None:
                    sampler.set_epoch(epoch)
                for b in loader:      # flip / rotation / scale drawn from Python's random, as the reference's transforms do
                    yield davis.to_device(b, device, augment=random, input_res=res, jpeg_status=jpeg_status, ids=ids)
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
        losses = training.parent_epoch(net, opt, bucket, epoch_batches(epoch), epoch, a.epochs, n_ave, state=loop_state,
                                       void=void)
        torch.cuda.synchronize()
        if jpeg_status is not None and int(jpeg_status) != 0:     # read after the epoch's synchronisation
            print(f"WARNING: rank {rank}: the device JPEG decoder flagged corrupt or cut-short frames in epoch {epoch} "
                  f"(status sum {int(jpeg_status)}); their bytes may differ from cv2.imread's")
            jpeg_status.zero_()
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
                                                                                   size_average=False, void=void)
                                        for o in outs])
                    if a.val_measures:
                        if stored:                   # the fused map at the annotation's own size (DESIGN.md §18)
                            g0 = s["gt_u8_stored"]
                            counts = measures(ops.resize_f32(outs[-1], g0.shape[1:]), g0)
                        else:
                            counts = measures(outs[-1], s["gt_u8"])
                        for i, fname in enumerate(s["fname"]):
                            per_seq.setdefault(fname.split("/")[0], evaluation.SequenceScores()).add(counts[i:i + 1])
            print("***Testing *** " + " ".join(f"Loss {k}: {v:.4f}" for k, v in enumerate((tot / len(val_batches)).tolist())))
            if a.val_measures:
                sc = evaluation.dataset_scores(per_seq)
                print("***Testing *** " + "  ".join(f"{m} M/O/D: {sc[m]['M']:.4f} / {sc[m]['O']:.4f} / {sc[m]['D']:.4f}"
                                                    for m in ("J", "F")) + f"  ({len(per_seq)} sequences)")
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
