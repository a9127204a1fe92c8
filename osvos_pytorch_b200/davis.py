"""DAVIS-2016 without the reference's ``dataloaders`` package: the host decodes, the device does the rest.

The reference's ``DAVIS2016`` dataset (dataloaders/davis_2016.py) decodes each frame with ``cv2.imread`` and then, in
a DataLoader worker, converts it to float32, subtracts the mean, normalises the mask, flips and warps both with cv2
and transposes them (``ToTensor``).  ``DAVIS2016Frames`` keeps the reference's file lists and decoder but stops at the
decoded bytes: an item is uint8 ``image`` [H,W,3] (BGR) and ``gt`` [H,W].  ``collate`` packs a batch into ONE uint8
buffer, so a ``DataLoader(..., collate_fn=collate)`` moves 4 bytes per pixel and ``to_device`` pins it and makes one
host-to-device copy of it.  There the ingest kernels (csrc/frames.cu) produce exactly the reference's float
tensors, or the fused warp produces the augmented ones (augment.affine_warp_u8).

``DeviceFrames`` decodes a whole split once and keeps the bytes on the device, so parent training decodes once per
run instead of once per epoch; each batch is then one indexed warp from the store (DESIGN.md §15).

``DAVIS2016Frames`` refuses ``inputRes``: its items are the decoded bytes at their stored size.  The reference's
``inputRes`` (``scipy.misc.imresize``, which no longer exists in SciPy) is a device stage here instead:
``input_res=`` on ``upload``, ``to_device``, ``DeviceFrames`` and ``inference.SequenceSegmenter`` resizes the image
(bilinear) and the mask (nearest) right after the upload, bit-identical to scipy 1.0's imresize (ops.resize_u8,
DESIGN.md §17), before the float conversion, flip and warp, the reference's order.  One deliberate difference: the
reference builds the all-zero mask of an unannotated frame at the stored size and never resizes it; here that mask
has the resized size, so that a batch has one size.
"""
import os
import random
import time

import numpy as np
import torch
from torch.utils.data import Dataset

from . import augment as _augment
from . import jpeg as _jpeg
from . import ops
from . import png as _png
from .evaluation import n_objects as _n_objects
from .ops import MEANVAL


def _cv2():
    try:
        import cv2
    except ImportError as e:
        raise ImportError("DAVIS2016Frames decodes frames with OpenCV (cv2.imread, the reference's decoder); "
                          "install opencv-python") from e
    return cv2


def default_db_root():
    return os.environ.get("OSVOS_DB_ROOT", "/path/to/DAVIS-2016")


class DAVIS2016Frames(Dataset):
    """The reference's DAVIS2016 file lists (dataloaders/davis_2016.py:31-64), items as decoded uint8 arrays.

    Without ``seq_name``: every frame of the sequences in ``train_seqs.txt`` (train) or ``val_seqs.txt``, with its
    annotation.  With ``seq_name``: the frames of that sequence, only the first one annotated (``train=True`` keeps
    just that first frame).  Items: ``image`` uint8 [H,W,3] BGR, ``gt`` uint8 [H,W] (zeros for a frame without an
    annotation), ``has_gt``, and ``fname`` = ``seq/%05d`` of the index in sequence mode (the reference's rule), else
    ``seq/<file stem>``.

    ``all_annotations=True`` (sequence mode): every frame carries its own annotation, as scoring the sequence needs; a
    sequence whose frame and annotation counts differ raises.

    ``decode="device"``: the worker reads the frame's file and parses its markers (jpeg.parse) instead of decoding it;
    the item carries ``jpeg`` (the parsed file) in place of ``image``, and ``collate`` / ``upload`` decode it on the
    device bit-identically to cv2.imread (ops.decode_jpeg, DESIGN.md §19).  A file outside the decoder's subset is
    decoded by cv2.imread as with ``decode="host"`` and carries ``image``.  Masks are decoded on the host either way."""

    def __init__(self, train=True, db_root_dir=None, seq_name=None, meanval=MEANVAL, inputRes=None,
                 all_annotations=False, decode="host"):
        if decode not in ("host", "device"):
            raise ValueError("decode must be 'host' or 'device'")
        self.decode = decode
        if inputRes is not None:
            raise NotImplementedError("inputRes: the reference resizes with scipy.misc.imresize, which SciPy no longer "
                                      "has, and neither entry point uses it; frames are read at their stored size")
        self.train, self.seq_name, self.meanval = train, seq_name, tuple(meanval)
        self.db_root_dir = default_db_root() if db_root_dir is None else db_root_dir
        root = self.db_root_dir
        split = "train_seqs" if train else "val_seqs"
        if seq_name is None:
            img_list, labels = [], []
            with open(os.path.join(root, split + ".txt")) as f:
                for seq in f.readlines():
                    seq = seq.strip()
                    images = np.sort(os.listdir(os.path.join(root, "JPEGImages/480p/", seq)))
                    img_list.extend(os.path.join("JPEGImages/480p/", seq, x) for x in images)
                    lab = np.sort(os.listdir(os.path.join(root, "Annotations/480p/", seq)))
                    labels.extend(os.path.join("Annotations/480p/", seq, x) for x in lab)
        else:
            names_img = np.sort(os.listdir(os.path.join(root, "JPEGImages/480p/", str(seq_name))))
            img_list = [os.path.join("JPEGImages/480p/", str(seq_name), x) for x in names_img]
            name_label = np.sort(os.listdir(os.path.join(root, "Annotations/480p/", str(seq_name))))
            if all_annotations:
                if len(name_label) != len(names_img):
                    raise ValueError(f"{root}: sequence {seq_name} has {len(names_img)} frames but {len(name_label)} "
                                     "annotations; scoring needs one per frame")
                labels = [os.path.join("Annotations/480p/", str(seq_name), x) for x in name_label]
            else:
                labels = [os.path.join("Annotations/480p/", str(seq_name), name_label[0])] + [None] * (len(names_img) - 1)
            if train:
                img_list, labels = [img_list[0]], [labels[0]]
        if len(labels) != len(img_list):
            raise ValueError(f"{root}: {len(img_list)} frames but {len(labels)} annotations in the {split} split")
        self.img_list, self.labels = img_list, labels

    def __len__(self):
        return len(self.img_list)

    def _read(self, rel, flags):
        cv2 = _cv2()
        arr = cv2.imread(os.path.join(self.db_root_dir, rel), flags)
        if arr is None:
            raise FileNotFoundError(f"cv2.imread could not read {os.path.join(self.db_root_dir, rel)}")
        return arr

    def _read_gt(self, rel):
        return self._read(rel, 0)

    def __getitem__(self, idx):
        item = {}
        parsed = None
        if self.decode == "device":
            with open(os.path.join(self.db_root_dir, self.img_list[idx]), "rb") as f:
                parsed = _jpeg.parse(f.read())
        if isinstance(parsed, _jpeg.Parsed):
            item["jpeg"] = parsed
            size = (parsed.h, parsed.w)
        else:
            item["image"] = self._read(self.img_list[idx], 1)          # cv2.IMREAD_COLOR: uint8 [H,W,3] BGR
            size = item["image"].shape[:2]
        has_gt = self.labels[idx] is not None
        gt = self._read_gt(self.labels[idx]) if has_gt else np.zeros(size, dtype=np.uint8)
        if self.seq_name is not None:
            fname = os.path.join(self.seq_name, "%05d" % idx)
        else:
            parts = self.img_list[idx].split("/")
            fname = os.path.join(parts[-2], os.path.splitext(parts[-1])[0])
        item.update(gt=gt, has_gt=has_gt, fname=fname)
        return item


class DAVIS2017Frames(DAVIS2016Frames):
    """DAVIS-2017 (semi-supervised), items as DAVIS2016Frames' with ``gt`` = the annotation's object ids and
    ``n_objects`` (DESIGN.md §24).

    The sequences are those of ``ImageSets/2017/<split>.txt`` (``split`` "train" or "val"), frames from
    ``JPEGImages/480p/<seq>/`` and annotations from ``Annotations/480p/<seq>/``, which are 8-bit palette PNGs: 0
    background, 1 .. K the objects, 255 void.  Each annotation is read as its indices (np.array(PIL.Image.open(f)), the
    toolkit's reader), never converted to gray.  A sequence's objects are 1 .. K with K = evaluation.n_objects of its
    first annotation, and ``palettes[seq]`` is that annotation's PLTE bytes (png.palette_of), the palette to write the
    sequence's results with.  ``seq_name`` and ``all_annotations`` are DAVIS2016Frames' sequence mode (only the first
    frame annotated unless ``all_annotations``); ``decode`` applies to the JPEG frames as there."""

    def __init__(self, split="val", db_root_dir=None, seq_name=None, all_annotations=False, decode="host"):
        if split not in ("train", "val"):
            raise ValueError("split must be 'train' or 'val'")
        if decode not in ("host", "device"):
            raise ValueError("decode must be 'host' or 'device'")
        self.decode, self.train, self.split, self.seq_name, self.meanval = decode, False, split, seq_name, MEANVAL
        self.db_root_dir = default_db_root() if db_root_dir is None else db_root_dir
        root = self.db_root_dir
        if seq_name is None:
            with open(os.path.join(root, "ImageSets", "2017", split + ".txt")) as f:
                seqs = [x.strip() for x in f if x.strip()]
        else:
            seqs = [str(seq_name)]
        img_list, labels, self.seq_of = [], [], []
        self.n_objects, self.palettes = {}, {}
        for seq in seqs:
            images = np.sort(os.listdir(os.path.join(root, "JPEGImages/480p/", seq)))
            anns = np.sort([x for x in os.listdir(os.path.join(root, "Annotations/480p/", seq)) if x.endswith(".png")])
            if not len(anns):
                raise ValueError(f"{root}: sequence {seq} has no annotation")
            if seq_name is None or all_annotations:
                if len(anns) != len(images):
                    raise ValueError(f"{root}: sequence {seq} has {len(images)} frames but {len(anns)} annotations")
                labs = [os.path.join("Annotations/480p/", seq, x) for x in anns]
            else:
                labs = [os.path.join("Annotations/480p/", seq, anns[0])] + [None] * (len(images) - 1)
            img_list.extend(os.path.join("JPEGImages/480p/", seq, x) for x in images)
            labels.extend(labs)
            self.seq_of.extend([seq] * len(images))
            with open(os.path.join(root, labs[0]), "rb") as f:
                first = f.read()
            self.n_objects[seq] = _n_objects(_png.decode_host_index(first))
            self.palettes[seq] = _png.palette_of(first)
        self.img_list, self.labels = img_list, labels

    def _read_gt(self, rel):
        with open(os.path.join(self.db_root_dir, rel), "rb") as f:
            return _png.decode_host_index(f.read())

    def __getitem__(self, idx):
        item = super().__getitem__(idx)
        item["n_objects"] = self.n_objects[self.seq_of[idx]]
        return item


def collate(items):
    """Items of one shape -> {'data': uint8 [N*H*W*4] (the N BGR frames, then the N masks), 'size': (N, H, W),
    'has_gt': bool [N], 'fname': [N]}.  One buffer, so pinning and the host-to-device copy are one transfer each.

    When any item carries ``jpeg`` (DAVIS2016Frames(decode="device")), 'data' holds instead the N masks, then the
    frames of the items that carry ``image``, then the packed JPEGs (jpeg.pack, 16-byte aligned), and 'jpeg' says
    which items are which (``upload`` assembles the frames on the device)."""
    h, w = items[0]["gt"].shape
    n = len(items)
    if any("jpeg" in it for it in items):
        return _collate_jpeg(items, n, h, w)
    data = torch.empty(n * h * w * 4, dtype=torch.uint8)
    img, gt = views(data, n, h, w)
    for i, it in enumerate(items):
        if it["image"].shape != (h, w, 3) or it["gt"].shape != (h, w):
            raise ValueError("all frames of a batch must share a size")
        img[i] = torch.from_numpy(it["image"])
        gt[i] = torch.from_numpy(it["gt"])
    return {"data": data, "size": torch.tensor([n, h, w]), "has_gt": torch.tensor([bool(it["has_gt"]) for it in items]),
            "fname": [it["fname"] for it in items]}


def _collate_jpeg(items, n, h, w):
    dec = [i for i, it in enumerate(items) if "jpeg" in it]
    fb = [i for i, it in enumerate(items) if "jpeg" not in it]
    for it in items:
        size = (it["jpeg"].h, it["jpeg"].w) if "jpeg" in it else it["image"].shape[:2]
        if tuple(size) != (h, w) or it["gt"].shape != (h, w):
            raise ValueError("all frames of a batch must share a size")
    blob = _jpeg.pack([items[i]["jpeg"] for i in dec])
    blob_off = -(-(n * h * w + len(fb) * h * w * 3) // 16) * 16
    data = torch.zeros(blob_off + len(blob), dtype=torch.uint8)
    gt = data[:n * h * w].view(n, h, w)
    img = data[n * h * w:n * h * w + len(fb) * h * w * 3].view(len(fb), h, w, 3)
    for i, it in enumerate(items):
        gt[i] = torch.from_numpy(it["gt"])
    for k, i in enumerate(fb):
        img[k] = torch.from_numpy(items[i]["image"])
    data[blob_off:] = torch.from_numpy(blob)
    return {"data": data, "size": torch.tensor([n, h, w]), "has_gt": torch.tensor([bool(it["has_gt"]) for it in items]),
            "fname": [it["fname"] for it in items],
            "jpeg": {"device": dec, "fallback": fb, "blob_off": blob_off, "nseg": _jpeg.segment_count(blob)}}


def _assemble(data, jp, n, h, w, jpeg_status=None, out=None):
    """The frames [N,H,W,3] (into ``out`` when given), masks [N,H,W] and status words int32 [N] (0 for host-decoded
    frames) of an uploaded JPEG batch (_collate_jpeg's layout): the packed JPEGs decoded on the device, the
    host-decoded frames copied into their slots.  ``jpeg_status``: an int32 [1] device tensor the status words are
    added to."""
    gt = data[:n * h * w].view(n, h, w)
    dec, fb = jp["device"], jp["fallback"]
    img = torch.empty((n, h, w, 3), dtype=torch.uint8, device=data.device) if out is None else out
    frame_status = torch.zeros(n, dtype=torch.int32, device=data.device)
    if fb:
        src = data[n * h * w:n * h * w + len(fb) * h * w * 3].view(len(fb), h, w, 3)
        if len(fb) == n:
            img.copy_(src)
        else:
            img[torch.tensor(fb, device=data.device)] = src
    if dec:
        blob = data[jp["blob_off"]:]
        out, status = ops.decode_jpeg(blob, len(dec), h, w, out=img if len(dec) == n else None, nseg=jp["nseg"])
        index = torch.tensor(dec, device=data.device)
        if len(dec) != n:
            img[index] = out
        frame_status[index] = status
        if jpeg_status is not None:
            jpeg_status += status.sum(dtype=torch.int32)
    return img, gt, frame_status


def device_views(batch, device, jpeg_status=None):
    """One host-to-device copy of a collated batch -> (image uint8 [N,H,W,3], gt uint8 [N,H,W], status int32 [N] or
    None) at the stored size: views of the copy, or for a decode="device" batch the frames decoded on the device
    (_assemble; status is the decoder's per frame, nonzero for a corrupt or cut-short stream)."""
    n, h, w = (int(v) for v in batch["size"])
    data = pinned(batch["data"]).to(device, non_blocking=True)
    if "jpeg" in batch:
        return _assemble(data, batch["jpeg"], n, h, w, jpeg_status)
    img, gt = views(data, n, h, w)
    return img, gt, None


def views(data, n, h, w):
    """The image [N,H,W,3] and mask [N,H,W] views of a collated buffer."""
    split = n * h * w * 3
    return data[:split].view(n, h, w, 3), data[split:split + n * h * w].view(n, h, w)


def pinned(data):
    """``data`` in page-locked memory, pinned in the calling thread.  Use this instead of a DataLoader's
    ``pin_memory=True``: the loader's pinning thread allocates page-locked memory at any moment, and such an allocation
    invalidates a CUDA graph the main thread is capturing (training steps and inference forwards are captured)."""
    return data if data.is_pinned() else data.pin_memory()


def imresize_size(size, h, w):
    """The (h', w') that scipy 1.0's ``imresize(arr, size)`` gives a frame of h x w (the reference's ``inputRes``): a
    tuple is (h', w'), an int is a percentage (int(dim * (size / 100.0))), a float a fraction (int(dim * size))."""
    if isinstance(size, (bool, np.bool_)):
        raise TypeError("input_res must be a (height, width) pair, an int percentage or a float fraction")
    if isinstance(size, (int, np.integer)):
        pct = int(size) / 100.0
        out = (int(h * pct), int(w * pct))
    elif isinstance(size, (float, np.floating)):
        out = (int(h * float(size)), int(w * float(size)))
    else:
        out = tuple(int(v) for v in size)
        if len(out) != 2:
            raise ValueError(f"input_res must be (height, width), got {size!r}")
    if min(out) < 1:
        raise ValueError(f"input_res {size!r} gives an empty frame {out} for a {h}x{w} frame")
    return out


def resize_pair(img, gt, input_res):
    """Device frames uint8 [N,H,W,3] and masks [N,H,W] at ``input_res`` (imresize_size): the image bilinear, the mask
    nearest, as the reference's make_img_gt_pair resizes them (dataloaders/davis_2016.py:96-99)."""
    h, w = (int(v) for v in img.shape[1:3])
    size = imresize_size(input_res, h, w)
    return ops.resize_u8(img, size, "bilinear"), ops.resize_u8(gt, size, "nearest")


def upload(batch, device, input_res=None, jpeg_status=None):
    """One host-to-device copy of a collated batch -> (image uint8 [N,H,W,3], gt uint8 [N,H,W], label stats).
    ``input_res``: the frames and masks are resized on the device first (resize_pair).  A batch of
    DAVIS2016Frames(decode="device") items is decoded on the device first (_assemble; ``jpeg_status``: an int32 [1]
    device tensor that accumulates the decoder's status words, nonzero when a stream was corrupt or cut short)."""
    img, gt, _ = device_views(batch, device, jpeg_status)
    if input_res is not None:
        img, gt = resize_pair(img, gt, input_res)
    return img, gt, ops.label_stats_u8(gt)


def to_device(batch, device, augment=None, meanval=MEANVAL, input_res=None, jpeg_status=None):
    """Collated batch -> {'image': f32 [N,3,H,W], 'gt': f32 [N,1,H,W]} on ``device``.

    augment None: the reference's make_img_gt_pair + ToTensor, bit for bit (ops.image_from_bgr8, ops.label_from_u8).
    Otherwise RandomHorizontalFlip + ScaleNRotate as the reference composes them, fused with the ingest
    (augment.affine_warp_u8): ``augment`` is a list of per-sample (flip, rot, scale) triples, or a random generator
    from which augment.draw_params draws them in the reference's order.  ``input_res``: the reference's ``inputRes``,
    applied on the device before all of that (upload, which also decodes a decode="device" batch's JPEGs)."""
    with torch.cuda.device(device):
        img, gt, stats = upload(batch, device, input_res, jpeg_status)
        if augment is None:
            return {"image": ops.image_from_bgr8(img, meanval), "gt": ops.label_from_u8(gt, stats)}
        params = augment if isinstance(augment, (list, tuple)) else _augment.draw_params(int(img.shape[0]), rng=augment)
        return _augment.affine_warp_u8(img, gt, params, stats, meanval)


_MAX_STATS_FRAMES = 65535                                # osvos_label_stats_u8 takes n < 65536


def shard(n, world, rank):
    """The dataset indices rank ``rank`` of ``world`` decodes for a DeviceFrames store: every world-th one, so each
    size group splits nearly evenly over the ranks and little padding is gathered."""
    return range(rank, n, world)


def shard_plan(sizes, world):
    """The store layout ``world`` ranks gather.  ``sizes``: (h, w) of every dataset index.  Returns one entry per size,
    in order of first appearance: ((h, w), pad, members), members[r] = the dataset indices of that size in rank r's
    shard, in decode order.  pad = the largest len(members[r]); rank r's share is sent as pad frames, so the gathered
    store has world * pad slots and member j of rank r sits in slot r * pad + j (the rest is padding)."""
    groups = {}
    for r in range(world):
        for i in shard(len(sizes), world, r):
            groups.setdefault(tuple(sizes[i]), [[] for _ in range(world)])[r].append(i)
    order = sorted(groups, key=lambda size: min(i for m in groups[size] for i in m))
    return [(size, max(len(m) for m in groups[size]), groups[size]) for size in order]


class DeviceFrames:
    """Every item of a DAVIS2016Frames, decoded once and kept on ``device`` as uint8 bytes.

    Frames are grouped by size; group g holds ``img`` uint8 [n_g,H,W,3], ``gt`` uint8 [n_g,H,W] and ``stats``
    (ops.label_stats_u8 of gt).  ``where[i]`` is dataset index i's (group, slot); ``has_gt`` and ``fname`` are the
    items' own.  A 480x854 frame takes 1.64 MB, so DAVIS-2016's train split (2,079 frames) takes 3.4 GB.

    The host decodes through a DataLoader(num_workers=workers, collate_fn=collate) in dataset order and holds its
    share until the device memory needed is known; the bytes are pinned in this thread (``pinned`` says why).  If
    they do not fit in torch.cuda.mem_get_info()'s free memory, ValueError is raised before anything is allocated.

    ``group``: a torch.distributed process group of R ranks.  Each rank then decodes a 1/R share (``shard``), the
    frame sizes are exchanged with all_gather_object, and the shares are gathered with NCCL all_gather_into_tensor,
    one call per size group and tensor, so every rank holds the whole store (layout: ``shard_plan``).

    ``input_res``: the reference's ``inputRes`` (imresize_size).  Each frame is resized on the device as it is stored
    (resize_pair), so the store, its size groups and the memory check are at the resized size; frames of different
    stored sizes that resize to one size share a group.  With a process group each rank resizes its own share before
    the gather.

    ``keep_stored_gt`` (with ``input_res``): the store also keeps every annotation's bytes at its stored size, in
    groups by stored size (``stored_groups``, each {'size', 'gt'}; ``where_stored[i]`` is index i's (group, slot)), so
    that segmentations upsampled back to that size (ops.resize_f32) are scored against the original annotations.  The
    memory check counts them, and ingest returns them as 'gt_u8_stored'.

    A ``decode="device"`` dataset's frames are decoded on the device (device_views).  Before the store is shared, every
    frame whose decoder status is nonzero (a corrupt or cut-short stream) is decoded again with cv2.imread, so the store
    holds cv2's bytes whatever the files.  ``fallback_frames``: frames outside the device decoder's subset (decoded by
    cv2.imread in the workers); ``redecoded_frames``: frames decoded again after a nonzero status."""

    def __init__(self, dataset, device, workers=0, group=None, input_res=None, keep_stored_gt=False):
        import torch.distributed as dist
        from torch.utils.data import DataLoader, Subset
        t0 = time.perf_counter()
        self.device = torch.device(device)
        world = 1 if group is None else dist.get_world_size(group)
        rank = 0 if group is None else dist.get_rank(group)
        n = len(dataset)
        mine = list(shard(n, world, rank))
        # a private generator: the loader's seed draw must not move the global RNG that training's samplers use
        loader = DataLoader(Subset(dataset, mine), batch_size=1, shuffle=False, num_workers=workers,
                            collate_fn=collate, generator=torch.Generator())
        decoded = dict(zip(mine, list(loader)))         # drained: the workers stop here, not in a finaliser
        meta = [(i, tuple(int(v) for v in b["size"][1:]), bool(b["has_gt"][0]), b["fname"][0])
                for i, b in decoded.items()]
        if group is not None:
            metas = [None] * world
            dist.all_gather_object(metas, meta, group=group)
            meta = sorted(m for ms in metas for m in ms)
        sizes = [m[1] if input_res is None else imresize_size(input_res, *m[1]) for m in meta]
        self.has_gt = [m[2] for m in meta]
        self.fname = [m[3] for m in meta]
        plan = shard_plan(sizes, world)
        keep_stored = keep_stored_gt and input_res is not None
        plan0 = shard_plan([m[1] for m in meta], world) if keep_stored else []
        need = sum(world * pad * (h * w * 4 + 8) for (h, w), pad, _ in plan)
        need += sum(world * pad * h * w for (h, w), pad, _ in plan0)
        free, _ = torch.cuda.mem_get_info(self.device)
        if need > free:
            raise ValueError(f"DeviceFrames: the {n} decoded frames need {need} bytes on {self.device} but only {free} "
                             "are free")
        self.groups, self.where = [], [None] * n
        self.stored_groups, self.where_stored = [], [None] * n
        self.fallback_frames = self.redecoded_frames = 0
        with torch.cuda.device(self.device):
            for g, ((h, w), pad, members) in enumerate(plan0):
                self.stored_groups.append({"size": (h, w), "gt": torch.zeros((world * pad, h, w), dtype=torch.uint8,
                                                                               device=self.device)})
                for r, m in enumerate(members):
                    for j, i in enumerate(m):
                        self.where_stored[i] = (g, r * pad + j)
            for g, ((h, w), pad, members) in enumerate(plan):
                img = torch.zeros((world * pad, h, w, 3), dtype=torch.uint8, device=self.device)
                gt = torch.zeros((world * pad, h, w), dtype=torch.uint8, device=self.device)
                checks = []
                for j, i in enumerate(members[rank]):
                    item = decoded.pop(i)
                    s = rank * pad + j
                    if "jpeg" not in item and getattr(dataset, "decode", "host") == "device":
                        self.fallback_frames += 1
                    if "jpeg" in item:
                        src_img, src_gt, st = device_views(item, self.device)
                        checks.append((i, s, st))
                    elif input_res is None:
                        src_img, src_gt = views(pinned(item["data"]), 1, h, w)
                    else:
                        h0, w0 = (int(v) for v in item["size"][1:])
                        src_img, src_gt = views(pinned(item["data"]).to(self.device, non_blocking=True), 1, h0, w0)
                    if input_res is None:
                        img[s].copy_(src_img[0], non_blocking=True)
                        gt[s].copy_(src_gt[0], non_blocking=True)
                    else:
                        ops.resize_u8(src_img, (h, w), "bilinear", out=img[s:s + 1])
                        ops.resize_u8(src_gt, (h, w), "nearest", out=gt[s:s + 1])
                        if keep_stored:
                            g0, s0 = self.where_stored[i]
                            self.stored_groups[g0]["gt"][s0].copy_(src_gt[0])
                if checks:                         # one synchronisation per size group, at build time only
                    flags = torch.cat([st for _, _, st in checks]).cpu()
                    for (i, s, _), f in zip(checks, flags.tolist()):
                        if f:
                            frame = torch.from_numpy(dataset._read(dataset.img_list[i], 1)).to(self.device)[None]
                            if input_res is None:
                                img[s:s + 1].copy_(frame)
                            else:
                                ops.resize_u8(frame, (h, w), "bilinear", out=img[s:s + 1])
                            self.redecoded_frames += 1
                if group is not None:              # in place: this rank's share is already in its slots
                    share = slice(rank * pad, (rank + 1) * pad)
                    dist.all_gather_into_tensor(img, img[share], group=group)
                    dist.all_gather_into_tensor(gt, gt[share], group=group)
                stats = torch.empty((world * pad, 2), dtype=torch.int32, device=self.device)
                for c0 in range(0, world * pad, _MAX_STATS_FRAMES):
                    stats[c0:c0 + _MAX_STATS_FRAMES] = ops.label_stats_u8(gt[c0:c0 + _MAX_STATS_FRAMES])
                self.groups.append({"size": (h, w), "img": img, "gt": gt, "stats": stats})
                for r, m in enumerate(members):
                    for j, i in enumerate(m):
                        self.where[i] = (g, r * pad + j)
            if group is not None:
                for (_, pad, _), grp in zip(plan0, self.stored_groups):
                    dist.all_gather_into_tensor(grp["gt"], grp["gt"][rank * pad:(rank + 1) * pad], group=group)
        torch.cuda.synchronize(self.device)
        self.nbytes = sum(t.numel() * t.element_size() for grp in self.groups for t in (grp["img"], grp["gt"], grp["stats"]))
        self.nbytes += sum(grp["gt"].numel() for grp in self.stored_groups)
        self.build_s = time.perf_counter() - t0

    def __len__(self):
        return len(self.where)

    def _slot(self, i):
        if not 0 <= i < len(self.where):
            raise IndexError(f"frame {i} outside a store of {len(self.where)} frames")
        return self.where[i]

    def augmented(self, indices, params):
        """The frames ``indices`` (dataset indices, one size), flipped and warped by ``params`` (one (flip, rot, scale)
        per frame) -> {'image': f32 [N,3,H,W], 'gt': f32 [N,1,H,W]}, bit-identical to
        to_device(collate(items), device, augment=params).  One indexed warp per 32 frames
        (augment.affine_warp_u8(index=...)); nothing is copied."""
        where = [self._slot(int(i)) for i in indices]
        g = where[0][0]
        if any(gi != g for gi, _ in where):
            raise ValueError("all frames of a batch must share a size")
        grp = self.groups[g]
        with torch.cuda.device(self.device):
            return _augment.affine_warp_u8(grp["img"], grp["gt"], params, grp["stats"], index=[s for _, s in where])

    def batches(self, index_batches, rng=random):
        """Augmented batches for an iterable of index batches (e.g. a DataLoader over dataset indices), the (flip, rot,
        scale) triples drawn from ``rng`` per batch as to_device(..., augment=rng) draws them."""
        for idx in index_batches:
            idx = [int(i) for i in idx]
            yield self.augmented(idx, _augment.draw_params(len(idx), rng=rng))

    def ingest(self, i):
        """Frame i without augmentation -> {'image': f32 [1,3,H,W], 'gt': f32 [1,1,H,W], 'gt_u8': uint8 [1,H,W] (a view
        of the store), 'fname': [name]}; image and gt are bit-identical to to_device(collate([item]), device).  A store
        built with keep_stored_gt adds 'gt_u8_stored': uint8 [1,H0,W0], the annotation at its stored size (a view)."""
        i = int(i)
        g, s = self._slot(i)
        grp = self.groups[g]
        gt = grp["gt"][s:s + 1]
        with torch.cuda.device(self.device):
            item = {"image": ops.image_from_bgr8(grp["img"][s:s + 1]), "gt": ops.label_from_u8(gt, grp["stats"][s:s + 1]),
                    "gt_u8": gt, "fname": [self.fname[i]]}
        if self.stored_groups:
            g0, s0 = self.where_stored[i]
            item["gt_u8_stored"] = self.stored_groups[g0]["gt"][s0:s0 + 1]
        return item
