#!/usr/bin/env python
"""Online (per-sequence) fine-tuning entry point - same role and defaults as the reference's
train_online.py: load the parent model, run nAveGrad x 2000 forward/backward passes on the annotated
first frame with SGD(lr 1e-8, momentum .9), save the weights, then segment the sequence.

    SEQ_NAME=blackswan python train_online.py --loader native # DAVIS on disk (needs cv2 + the dataset)
    SEQ_NAME=blackswan python train_online.py --loader native --evaluate   # ... and score the masks (J and F)
    SEQ_NAME=dogs-jump python train_online.py --loader native --davis 2017 --evaluate   # DAVIS-2017, one net per object
    SEQ_NAME=dogs-jump python train_online.py --loader native --davis 2017 --input-res 240 427 --output-res stored
    SEQ_NAME=blackswan python train_online.py                 # the same through the reference's dataloaders package
    python train_online.py --synthetic --iters 200            # synthetic 480x854 frame, no dataset

Single GPU by design (BASELINE.json: online fine-tune stays single-GPU; run one sequence per GPU)."""
import argparse
import os
import timeit

import collections

import numpy as np
import torch

import networks.vgg_osvos as vo
from mypath import Path
from osvos_pytorch_b200 import ops, training


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
    ap.add_argument("--upsampling-lr", type=float, default=0.0,
                    help="lr of the side-output deconvolutions (upscale / upscale_); 0 keeps them fixed as the reference "
                         "does, a nonzero value trains them (the net learns its upsampling)")
    ap.add_argument("--deterministic", action="store_true",
                    help="torch.use_deterministic_algorithms(True) before anything is built: the package's kernels "
                         "reduce in a fixed order, so two runs on the same device give bit-identical results")
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
    ap.add_argument("--decode", default="host", choices=["host", "device"],
                    help="--loader native: decode the JPEG frames with cv2.imread in the workers (host), or parse them "
                         "there and decode them on the GPU, bit-identically (device; files outside the decoder's subset "
                         "still go through cv2.imread)")
    ap.add_argument("--input-res", type=int, nargs=2, default=None, metavar=("H", "W"),
                    help="the reference's inputRes: resize every frame (bilinear) and annotation (nearest) to H x W on "
                         "the device before training, segmentation and scoring, as scipy 1.0's imresize does. Needs "
                         "--loader native (--synthetic has --height / --width); with --davis 2017 it needs "
                         "--output-res stored")
    ap.add_argument("--output-res", default="network", choices=["network", "stored"],
                    help="with --input-res: write (and with --evaluate score) the masks at the network resolution H x W "
                         "(network), or at each frame's stored size (stored): the fused logits are upsampled on the "
                         "device as scipy 1.0's imresize(mode='F') does and scored against the original annotations, "
                         "so the PNGs and J / F compare with the DAVIS-2016 benchmark's. With --davis 2017 each "
                         "object's logits are upsampled and then merged into the stored-size label map in one kernel "
                         "(ops.upsample_merge_objects). Without --input-res it changes nothing")
    ap.add_argument("--encode", default="host", choices=["host", "device"],
                    help="write the result PNGs with Pillow on the host (host), or encode them on the GPU "
                         "(device: SequenceSegmenter(encode='png'); the bytes are written as they come, no Pillow)")
    ap.add_argument("--overlay", action="store_true",
                    help="also write each frame with its mask drawn over it (the reference's vis_res picture: the "
                         "foreground blended 50/50 with red, its outline black) as Results/<seq>_overlay/<frame>.jpg, "
                         "drawn and JPEG-encoded on the GPU (the bytes cv2.imwrite would write). Needs --loader native. "
                         "With --davis 2017 each object is drawn in its palette colour with its own outline, from the "
                         "written label files (visualize.render_results)")
    ap.add_argument("--overlay-quality", type=int, default=95, help="JPEG quality of --overlay (1..100)")
    ap.add_argument("--davis", default="2016", choices=["2016", "2017"],
                    help="2017: a DAVIS-2017 sequence (palette annotations of K objects). The parent is fine-tuned once "
                         "per object on the first frame with that object's mask, every frame goes through the K nets "
                         "and each pixel takes the object of the largest positive fused logit; the results are palette "
                         "PNGs of object ids (the first annotation's palette) and --evaluate scores every object. "
                         "Needs --loader native; K fine-tunes take K times as long. --input-res H W --output-res stored "
                         "fine-tunes and segments at H x W and writes and scores the label maps at the stored size")
    ap.add_argument("--ignore-void", action="store_true",
                    help="with --davis 2017: leave the annotation's void pixels (255) out of each object's fine-tuning "
                         "loss instead of counting them as background. Needs a parent whose deconvolution weights are "
                         "the bilinear taps (not one trained with --upsampling-lr)")
    a = ap.parse_args(argv)
    if a.ignore_void and a.davis != "2017":
        ap.error("--ignore-void applies to --davis 2017 (DAVIS-2016 annotations have no void pixels)")
    if a.ignore_void and a.upsampling_lr != 0.0:
        ap.error("--ignore-void trains with void labels, which the learned-upsampling tail does not support; it cannot "
                 "be combined with a nonzero --upsampling-lr")
    if a.evaluate and (a.synthetic or a.loader != "native"):
        ap.error("--evaluate scores against the DAVIS annotations read by --loader native; it cannot be combined with "
                 + ("--synthetic" if a.synthetic else "--loader reference"))
    if a.input_res is not None and (a.synthetic or a.loader != "native"):
        ap.error("--input-res resizes the frames read by --loader native; it cannot be combined with "
                 + ("--synthetic (use --height / --width)" if a.synthetic else "--loader reference"))
    if a.decode == "device" and (a.synthetic or a.loader != "native"):
        ap.error("--decode device decodes the frames read by --loader native; it cannot be combined with "
                 + ("--synthetic" if a.synthetic else "--loader reference"))
    if a.overlay and (a.synthetic or a.loader != "native"):
        ap.error("--overlay draws over the frames read by --loader native; it cannot be combined with "
                 + ("--synthetic" if a.synthetic else "--loader reference"))
    if not 1 <= a.overlay_quality <= 100:
        ap.error("--overlay-quality must lie in 1..100")
    if a.davis == "2017":
        if a.synthetic or a.loader != "native":
            ap.error("--davis 2017 reads the sequence with --loader native; it cannot be combined with "
                     + ("--synthetic" if a.synthetic else "--loader reference"))
        if a.input_res is not None and a.output_res != "stored":
            ap.error("--davis 2017 writes label maps at the stored size: --input-res needs --output-res stored")
    return a


def main(argv=None):
    a = parse(argv)
    if a.deterministic:
        torch.use_deterministic_algorithms(True)
    iters = a.iters if a.iters is not None else 2000 * a.n_ave_grad
    if a.lr is None:
        a.lr = 1e-10 if a.synthetic else 1e-8
    log_every = a.log_every if a.log_every is not None else max(1, iters // 20)
    save_dir = Path.save_root_dir()
    os.makedirs(save_dir, exist_ok=True)
    device = torch.device(f"cuda:{a.gpu_id}")
    torch.cuda.set_device(device)

    net = vo.OSVOS(pretrained=0, precision=a.precision, learn_upsampling=a.upsampling_lr != 0.0)
    if a.synthetic:
        vo.he_init_(net, seed=a.seed)
        with torch.no_grad():               # keep the synthetic logits O(10): scale the side branch down
            for mod in list(net.side_prep) + [net.fuse]:
                mod.weight.mul_(0.1)
    else:
        ckpt = os.path.join(save_dir, f"{a.parent_name}_epoch-{a.parent_epoch - 1}.pth")
        net.load_state_dict(torch.load(ckpt, map_location="cpu"))
    if a.davis == "2017":
        return online_2017(a, net.state_dict(), device, save_dir, iters, log_every)
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
        first = davis.DAVIS2016Frames(train=True, db_root_dir=Path.db_root_dir(), seq_name=a.seq_name, decode=a.decode)
        input_res = None if a.input_res is None else tuple(a.input_res)
        img_u8, gt_u8, stats = davis.upload(davis.collate([first[0]]), device, input_res=input_res)
        rng = random.Random(a.seed)

        def sample_fn(it):
            return augment.affine_warp_u8(img_u8, gt_u8, augment.draw_params(1, rng=rng), stats)
        db_test = davis.DAVIS2016Frames(train=False, db_root_dir=Path.db_root_dir(), seq_name=a.seq_name,
                                        all_annotations=a.evaluate, decode=a.decode)
        # pinned here, between forwards, not by a loader thread that could allocate during a graph capture; the image
        # and the mask are two views of the one pinned buffer
        test_loader = DataLoader(db_test, batch_size=1, shuffle=False, num_workers=1, collate_fn=davis.collate)
        if a.decode == "device":         # collated batches as they are: the segmenter decodes them on the device
            test_frames = test_loader
        else:
            test_frames = (dict(zip(("image", "gt"), davis.views(davis.pinned(b["data"]), *(int(v) for v in b["size"]))),
                                fname=b["fname"]) for b in test_loader)
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
    history = training.online_finetune(net, sample_fn, iters, a.n_ave_grad, a.lr, a.wd, log_every,
                                       upsampling_lr=a.upsampling_lr)
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
    from osvos_pytorch_b200.inference import SequenceSegmenter
    names = collections.deque()
    native = a.loader == "native" and not a.synthetic
    input_res = None if a.input_res is None else tuple(a.input_res)
    upsample = input_res is not None and a.output_res == "stored"
    stored_hw = []                                      # the sequence's stored size (one size per sequence)

    jpeg_frames = native and a.decode == "device"

    def frames():
        for ii, s in enumerate(test_frames):
            shape = tuple(int(v) for v in s["size"]) if jpeg_frames else tuple(s["image"].shape[:3])   # N, H, W
            names.append([os.path.basename(s["fname"][jj]) if "fname" in s else f"{ii:05d}_{jj}"
                          for jj in range(shape[0])])
            if upsample and not stored_hw:
                stored_hw.extend(shape[1:3])
            if jpeg_frames:                 # a collated batch: the segmenter takes the masks from it
                yield s
            else:
                yield (s["image"], s["gt"]) if a.evaluate else s["image"]
    if upsample:
        print(f"Frames resized to {input_res[0]}x{input_res[1]} (inputRes); the fused logits are upsampled to the "
              "stored size, results are written at that size"
              + (", scored against the original annotations" if a.evaluate else ""))
    elif input_res is not None:
        print(f"Frames resized to {input_res[0]}x{input_res[1]} (inputRes); results are written at that size"
              + (", scored against the nearest-resized annotations" if a.evaluate else ""))
    seg = SequenceSegmenter(net, output="bytescale", frames=("jpeg" if jpeg_frames else "bgr8") if native else "nchw_f32",
                            score=a.evaluate,
                            input_res=input_res, output_res=a.output_res,
                            encode="png" if a.encode == "device" else None,
                            overlay="jpeg" if a.overlay else None, overlay_quality=a.overlay_quality)
    if a.overlay:
        overlay_dir = os.path.join(save_dir, "Results", a.seq_name + "_overlay")
        os.makedirs(overlay_dir, exist_ok=True)
    for pred in seg(frames()):
        batch_names = names.popleft()
        if a.overlay:                                   # one complete JPEG file per frame
            pred, overlays = pred
            for jj, name in enumerate(batch_names):
                with open(os.path.join(overlay_dir, name + ".jpg"), "wb") as f:
                    f.write(overlays[jj])
        if a.encode == "device":                        # one complete PNG file per frame
            for jj, name in enumerate(batch_names):
                with open(os.path.join(out_dir, name + ".png"), "wb") as f:
                    f.write(pred[jj])
            continue
        arr = pred.numpy()
        for jj, name in enumerate(batch_names):
            try:
                from PIL import Image
                Image.fromarray(arr[jj, 0], mode="L").save(os.path.join(out_dir, name + ".png"))
            except ImportError:
                np.save(os.path.join(out_dir, name + ".npy"), arr[jj, 0])
    if seg.jpeg_status is not None and int(seg.jpeg_status) != 0:     # the segmenter's last wait covered the decodes
        print(f"WARNING: the device JPEG decoder flagged corrupt or cut-short frames (status sum {int(seg.jpeg_status)}); "
              "their bytes may differ from cv2.imread's")
    if a.evaluate:
        import json
        from osvos_pytorch_b200.evaluation import SequenceScores
        scores = SequenceScores()
        scores.add(seg.frame_counts())
        res = scores.result()
        st = res["statistics"]
        print("Scores of " + a.seq_name + " (frames 1 .. n-2): "
              + "  ".join(f"{m} M/O/D: {st[m]['M']:.4f} / {st[m]['O']:.4f} / {st[m]['D']:.4f}" for m in ("J", "F")))
        if upsample:
            res = dict(network_res=list(input_res), scored_res=stored_hw, **res)
        with open(os.path.join(save_dir, "Results", a.seq_name + "_scores.json"), "w") as f:
            json.dump(dict(sequence=a.seq_name, **res), f, indent=1)
    return history


def online_2017(a, parent, device, save_dir, iters, log_every):
    """DAVIS-2017 semi-supervised (DESIGN.md §24): one fine-tune of the parent weights ``parent`` per object of the
    first annotation, then the sequence segmented by the K nets and merged into label maps."""
    import json
    import random
    from torch.utils.data import DataLoader
    from osvos_pytorch_b200 import augment, davis
    from osvos_pytorch_b200.evaluation import ObjectScores
    from osvos_pytorch_b200.inference import SequenceSegmenter
    first_ds = davis.DAVIS2017Frames(db_root_dir=Path.db_root_dir(), seq_name=a.seq_name, decode=a.decode)
    first = first_ds[0]                              # read once: every object trains on these bytes
    k_objects, palette = first["n_objects"], first_ds.palettes[a.seq_name]
    if k_objects < 1:
        raise SystemExit(f"sequence {a.seq_name}: the first annotation has no object")
    input_res = None if a.input_res is None else tuple(a.input_res)
    # the image bilinear, the id map nearest (ids survive): every object fine-tunes at the network resolution
    img_u8, ids_u8, _ = davis.upload(davis.collate([first]), device, input_res=input_res)
    if a.ignore_void:                                # refused before any fine-tune starts, not at its first step
        probe = vo.OSVOS(pretrained=0, precision=a.precision, verbose=False)
        probe.load_state_dict(parent)
        if probe._engine.uses_general_tail():
            raise SystemExit("--ignore-void: the parent's deconvolution weights are not the bilinear taps, and void "
                             "labels are not supported by the general tail they need")
    print(f"Start of Online Training, sequence: {a.seq_name}, {k_objects} object(s)")
    nets, history = [], []
    t0 = timeit.default_timer()
    for k in range(1, k_objects + 1):
        net = vo.OSVOS(pretrained=0, precision=a.precision, learn_upsampling=a.upsampling_lr != 0.0)
        net.load_state_dict(parent)
        net.to(device)
        rng = random.Random(a.seed)
        if a.ignore_void:                            # id == k -> 1, 255 -> void, else 0 (the warp's id mode)
            def sample_fn(it, k=k, rng=rng):
                return augment.affine_warp_u8(img_u8, ids_u8, augment.draw_params(1, rng=rng), ids=k)
        else:
            gt_k = torch.where(ids_u8 == k, 255, 0).to(torch.uint8)      # the object's binary mask as 0 / 255 bytes
            stats_k = ops.label_stats_u8(gt_k)

            def sample_fn(it, gt_k=gt_k, stats_k=stats_k, rng=rng):
                return augment.affine_warp_u8(img_u8, gt_k, augment.draw_params(1, rng=rng), stats_k)
        hist = training.online_finetune(net, sample_fn, iters, a.n_ave_grad, a.lr, a.wd, log_every,
                                        upsampling_lr=a.upsampling_lr, void=a.ignore_void)
        if hist and not all(v == v and abs(v) != float("inf") for v in hist):
            print(f"WARNING: object {k}: non-finite loss - lower --lr for this initialisation")
        history.append(hist)
        if not a.no_save:
            torch.save(net.state_dict(), os.path.join(save_dir, f"{a.seq_name}_object-{k}_epoch-{iters - 1}.pth"))
        net.eval()
        nets.append(net)
    torch.cuda.synchronize()
    dt = timeit.default_timer() - t0
    print(f"Online training time: {dt:.2f} s for {k_objects} object(s) ({k_objects * iters / dt:.1f} fwd+bwd/s)")

    print("Testing Network")
    out_dir = os.path.join(save_dir, "Results", a.seq_name)
    os.makedirs(out_dir, exist_ok=True)
    db_test = davis.DAVIS2017Frames(db_root_dir=Path.db_root_dir(), seq_name=a.seq_name, all_annotations=a.evaluate,
                                    decode=a.decode)
    test_loader = DataLoader(db_test, batch_size=1, shuffle=False, num_workers=1, collate_fn=davis.collate)
    jpeg_frames = a.decode == "device"
    names = collections.deque()
    stored_hw = []                                      # the sequence's stored size (one size per sequence)

    def frames():
        for b in test_loader:
            names.append([os.path.basename(f) for f in b["fname"]])
            if not stored_hw:
                stored_hw.extend(int(v) for v in b["size"][1:3])
            if jpeg_frames:
                yield b
            else:
                img, gt = davis.views(davis.pinned(b["data"]), *(int(v) for v in b["size"]))
                yield (img, gt) if a.evaluate else img
    encode = a.encode == "device"
    if input_res is not None:
        print(f"Frames resized to {input_res[0]}x{input_res[1]} (inputRes); each object's fused logits are upsampled to "
              "the stored size and merged there, label maps are written at that size"
              + (", scored against the original annotations" if a.evaluate else ""))
    seg = SequenceSegmenter(nets=nets, output="labels", frames="jpeg" if jpeg_frames else "bgr8", score=a.evaluate,
                            input_res=input_res, output_res=a.output_res,
                            encode="png" if encode else None, palette=palette if encode else None)
    for pred in seg(frames()):
        batch_names = names.popleft()
        for jj, name in enumerate(batch_names):
            path = os.path.join(out_dir, name + ".png")
            if encode:                                  # one complete palette PNG file per frame
                with open(path, "wb") as f:
                    f.write(pred[jj])
            else:
                from PIL import Image
                im = Image.fromarray(pred.numpy()[jj, 0], mode="P")
                if palette is not None:
                    im.putpalette(palette)
                im.save(path)
    if seg.jpeg_status is not None and int(seg.jpeg_status) != 0:
        print(f"WARNING: the device JPEG decoder flagged corrupt or cut-short frames (status sum {int(seg.jpeg_status)})")
    if a.overlay:                                       # drawn from the label files just written, on the device
        from osvos_pytorch_b200 import visualize
        visualize.render_results(os.path.join(save_dir, "Results"), Path.db_root_dir(), sequences=[a.seq_name],
                                 davis="2017", quality=a.overlay_quality, device=device, decode=a.decode,
                                 palette=palette)
    if a.evaluate:
        scores = ObjectScores(k_objects)
        scores.add(seg.frame_counts())
        res = scores.result()
        if input_res is not None:
            res = dict(network_res=list(input_res), scored_res=stored_hw, **res)
        for k, ob in res["objects"].items():
            st = ob["statistics"]
            print(f"Scores of {a.seq_name} object {k} (frames 1 .. n-2): "
                  + "  ".join(f"{m} M/O/D: {st[m]['M']:.4f} / {st[m]['O']:.4f} / {st[m]['D']:.4f}" for m in ("J", "F")))
        with open(os.path.join(save_dir, "Results", a.seq_name + "_scores.json"), "w") as f:
            json.dump(dict(sequence=a.seq_name, davis="2017", n_objects=k_objects, **res), f, indent=1)
    return history


if __name__ == "__main__":
    main()
