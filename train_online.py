#!/usr/bin/env python
"""Online (per-sequence) fine-tuning entry point - same role and defaults as the reference's
train_online.py: load the parent model, run nAveGrad x 2000 forward/backward passes on the annotated
first frame with SGD(lr 1e-8, momentum .9), save the weights, then segment the sequence.

    SEQ_NAME=blackswan python train_online.py --loader native # DAVIS on disk (needs cv2 + the dataset)
    SEQ_NAME=blackswan python train_online.py --loader native --evaluate   # ... and score the masks (J and F)
    SEQ_NAME=blackswan python train_online.py                 # the same through the reference's dataloaders package
    python train_online.py --synthetic --iters 200            # synthetic 480x854 frame, no dataset

Single GPU by design (BASELINE.json: online fine-tune stays single-GPU; run one sequence per GPU)."""
import argparse
import os
import timeit

import numpy as np
import torch

import networks.vgg_osvos as vo
from mypath import Path
from osvos_pytorch_b200 import training


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--seq-name", default=os.environ.get("SEQ_NAME", "blackswan"))
    ap.add_argument("--n-ave-grad", type=int, default=5)
    ap.add_argument("--iters", type=int, default=None, help="forward/backward passes (default 2000 * nAveGrad)")
    ap.add_argument("--parent-epoch", type=int, default=240)
    ap.add_argument("--parent-name", default="parent")
    ap.add_argument("--lr", type=float, default=None, help="default 1e-8 (reference); 1e-10 with --synthetic, whose "
                    "He-initialised network produces O(10)-scale logits and therefore much larger summed-loss gradients")
    ap.add_argument("--wd", type=float, default=0.0002)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--gpu-id", type=int, default=0)
    ap.add_argument("--precision", default="exact", choices=["exact", "fast"])
    ap.add_argument("--synthetic", action="store_true", help="synthetic frame + He-init weights instead of DAVIS + parent model")
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=854)
    ap.add_argument("--log-every", type=int, default=None)
    ap.add_argument("--no-save", action="store_true")
    ap.add_argument("--gpu-augment", action="store_true",
                    help="RandomHorizontalFlip + ScaleNRotate on the device (osvos_pytorch_b200.augment) on the "
                         "GPU-resident annotated frame instead of cv2 in a DataLoader worker")
    ap.add_argument("--loader", default="reference", choices=["reference", "native"],
                    help="real data: the reference's dataloaders package (reference), or osvos_pytorch_b200.davis "
                         "(native: cv2 decodes, the device ingests and augments; the augmentation is always on the "
                         "device)")
    ap.add_argument("--evaluate", action="store_true",
                    help="score the segmentation against every frame's annotation on the device (DAVIS-2016 J and F, "
                         "osvos_pytorch_b200.evaluation); prints them and writes Results/<seq>_scores.json. "
                         "Needs --loader native")
    a = ap.parse_args(argv)
    if a.evaluate and (a.synthetic or a.loader != "native"):
        ap.error("--evaluate scores against the DAVIS annotations read by --loader native; it cannot be combined with "
                 + ("--synthetic" if a.synthetic else "--loader reference"))
    return a


def main(argv=None):
    a = parse(argv)
    iters = a.iters if a.iters is not None else 2000 * a.n_ave_grad
    if a.lr is None:
        a.lr = 1e-10 if a.synthetic else 1e-8
    log_every = a.log_every if a.log_every is not None else max(1, iters // 20)
    save_dir = Path.save_root_dir()
    os.makedirs(save_dir, exist_ok=True)
    device = torch.device(f"cuda:{a.gpu_id}")
    torch.cuda.set_device(device)

    net = vo.OSVOS(pretrained=0, precision=a.precision)
    if a.synthetic:
        vo.he_init_(net, seed=a.seed)
        with torch.no_grad():               # keep the synthetic logits O(10): scale the side branch down
            for mod in list(net.side_prep) + [net.fuse]:
                mod.weight.mul_(0.1)
    else:
        ckpt = os.path.join(save_dir, f"{a.parent_name}_epoch-{a.parent_epoch - 1}.pth")
        net.load_state_dict(torch.load(ckpt, map_location="cpu"))
    net.to(device)

    if a.synthetic:
        fixed = training.synthetic_batch(1, a.height, a.width, 1234 + a.seed, device)

        if a.gpu_augment:
            import random
            from osvos_pytorch_b200 import augment
            rng = random.Random(a.seed)

            def sample_fn(it):
                return augment.augment_batch(fixed, rng=rng)
        else:
            def sample_fn(it):
                return fixed
        test_frames = [fixed]
    elif a.loader == "native":
        # the annotated frame is decoded once and stays on the device as bytes; every iteration draws a flip, rotation
        # and scale (the reference's order) and the fused warp ingests and augments it in one pass
        import random
        from torch.utils.data import DataLoader
        from osvos_pytorch_b200 import augment, davis
        first = davis.DAVIS2016Frames(train=True, db_root_dir=Path.db_root_dir(), seq_name=a.seq_name)
        img_u8, gt_u8, stats = davis.upload(davis.collate([first[0]]), device)
        rng = random.Random(a.seed)

        def sample_fn(it):
            return augment.affine_warp_u8(img_u8, gt_u8, augment.draw_params(1, rng=rng), stats)
        db_test = davis.DAVIS2016Frames(train=False, db_root_dir=Path.db_root_dir(), seq_name=a.seq_name,
                                        all_annotations=a.evaluate)
        # pinned here, between forwards, not by a loader thread that could allocate during a graph capture; the image
        # and the mask are two views of the one pinned buffer
        test_frames = (dict(zip(("image", "gt"), davis.views(davis.pinned(b["data"]), *(int(v) for v in b["size"]))),
                            fname=b["fname"])
                       for b in DataLoader(db_test, batch_size=1, shuffle=False, num_workers=1, collate_fn=davis.collate))
    else:
        from dataloaders import davis_2016 as db
        from dataloaders import custom_transforms as tr
        from torch.utils.data import DataLoader
        from torchvision import transforms
        aug = transforms.Compose([tr.RandomHorizontalFlip(), tr.ScaleNRotate(rots=(-30, 30), scales=(.75, 1.25)),
                                  tr.ToTensor()])
        db_train = db.DAVIS2016(train=True, db_root_dir=Path.db_root_dir(), transform=aug, seq_name=a.seq_name)
        db_test = db.DAVIS2016(train=False, db_root_dir=Path.db_root_dir(), transform=tr.ToTensor(), seq_name=a.seq_name)
        loader = DataLoader(db_train, batch_size=1, shuffle=True, num_workers=1, persistent_workers=True)
        state = {"it": iter(loader)}
        if a.gpu_augment:
            # the online set is the single annotated frame (train=True with seq_name): keep it on the GPU and draw a
            # fresh flip / rotation / scale per iteration there
            import random
            from osvos_pytorch_b200 import augment
            raw = db.DAVIS2016(train=True, db_root_dir=Path.db_root_dir(), transform=tr.ToTensor(), seq_name=a.seq_name)[0]
            base = {"image": raw["image"][None].to(device), "gt": raw["gt"][None].to(device)}
            rng = random.Random(a.seed)

        def sample_fn(it):
            if a.gpu_augment:
                return augment.augment_batch(base, rng=rng)
            np.random.seed(a.seed + it)
            try:
                s = next(state["it"])
            except StopIteration:
                state["it"] = iter(loader)
                s = next(state["it"])
            return {"image": s["image"].to(device, non_blocking=True), "gt": s["gt"].to(device, non_blocking=True)}
        test_frames = DataLoader(db_test, batch_size=1, shuffle=False, num_workers=1)

    print("Start of Online Training, sequence: " + a.seq_name)
    t0 = timeit.default_timer()
    history = training.online_finetune(net, sample_fn, iters, a.n_ave_grad, a.lr, a.wd, log_every)
    torch.cuda.synchronize()
    dt = timeit.default_timer() - t0
    print(f"Online training time: {dt:.2f} s ({iters / dt:.1f} fwd+bwd/s, {iters / a.n_ave_grad / dt:.1f} SGD steps/s)")
    if history and not all(v == v and abs(v) != float("inf") for v in history):
        print("WARNING: non-finite loss - lower --lr for this initialisation")
    if not a.no_save:
        torch.save(net.state_dict(), os.path.join(save_dir, f"{a.seq_name}_epoch-{iters - 1}.pth"))

    print("Testing Network")
    out_dir = os.path.join(save_dir, "Results", a.seq_name)
    os.makedirs(out_dir, exist_ok=True)
    net.eval()
    # The reference's test loop (train_online.py:172-187): forward -> numpy sigmoid -> scipy.misc.imsave, which min-max
    # bytescales each frame.  Same payload here, produced on the device (ops.logits_to_u8 mode "bytescale") with the
    # H2D / forward / D2H legs of consecutive frames overlapped (inference.SequenceSegmenter).
    import collections
    from osvos_pytorch_b200.inference import SequenceSegmenter
    names = collections.deque()

    def frames():
        for ii, s in enumerate(test_frames):
            n = int(s["image"].shape[0])
            names.append([os.path.basename(s["fname"][jj]) if "fname" in s else f"{ii:05d}_{jj}" for jj in range(n)])
            yield (s["image"], s["gt"]) if a.evaluate else s["image"]
    native = a.loader == "native" and not a.synthetic
    seg = SequenceSegmenter(net, output="bytescale", frames="bgr8" if native else "nchw_f32", score=a.evaluate)
    for pred in seg(frames()):
        arr = pred.numpy()
        for jj, name in enumerate(names.popleft()):
            try:
                from PIL import Image
                Image.fromarray(arr[jj, 0], mode="L").save(os.path.join(out_dir, name + ".png"))
            except ImportError:
                np.save(os.path.join(out_dir, name + ".npy"), arr[jj, 0])
    if a.evaluate:
        import json
        from osvos_pytorch_b200.evaluation import SequenceScores
        scores = SequenceScores()
        scores.add(seg.frame_counts())
        res = scores.result()
        st = res["statistics"]
        print("Scores of " + a.seq_name + " (frames 1 .. n-2): "
              + "  ".join(f"{m} M/O/D: {st[m]['M']:.4f} / {st[m]['O']:.4f} / {st[m]['D']:.4f}" for m in ("J", "F")))
        with open(os.path.join(save_dir, "Results", a.seq_name + "_scores.json"), "w") as f:
            json.dump(dict(sequence=a.seq_name, **res), f, indent=1)
    return history


if __name__ == "__main__":
    main()
