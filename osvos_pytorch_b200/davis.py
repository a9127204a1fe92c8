"""DAVIS-2016 without the reference's ``dataloaders`` package: the host decodes, the device does the rest.

The reference's ``DAVIS2016`` dataset (dataloaders/davis_2016.py) decodes each frame with ``cv2.imread`` and then, in
a DataLoader worker, converts it to float32, subtracts the mean, normalises the mask, flips and warps both with cv2
and transposes them (``ToTensor``).  ``DAVIS2016Frames`` keeps the reference's file lists and decoder but stops at the
decoded bytes: an item is uint8 ``image`` [H,W,3] (BGR) and ``gt`` [H,W].  ``collate`` packs a batch into ONE uint8
buffer, so a ``DataLoader(..., collate_fn=collate)`` moves 4 bytes per pixel and ``to_device`` pins it and makes one
host-to-device copy of it.  There the ingest kernels (csrc/frames.cu) produce exactly the reference's float
tensors, or the fused warp produces the augmented ones (augment.affine_warp_u8).

``inputRes`` is not supported: the reference resizes with ``scipy.misc.imresize``, which no longer exists in SciPy, and
neither entry point sets it.
"""
import os

import numpy as np
import torch
from torch.utils.data import Dataset

from . import augment as _augment
from . import ops
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
    sequence whose frame and annotation counts differ raises."""

    def __init__(self, train=True, db_root_dir=None, seq_name=None, meanval=MEANVAL, inputRes=None,
                 all_annotations=False):
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

    def __getitem__(self, idx):
        image = self._read(self.img_list[idx], 1)                      # cv2.IMREAD_COLOR: uint8 [H,W,3] BGR
        has_gt = self.labels[idx] is not None
        gt = self._read(self.labels[idx], 0) if has_gt else np.zeros(image.shape[:2], dtype=np.uint8)
        if self.seq_name is not None:
            fname = os.path.join(self.seq_name, "%05d" % idx)
        else:
            parts = self.img_list[idx].split("/")
            fname = os.path.join(parts[-2], os.path.splitext(parts[-1])[0])
        return {"image": image, "gt": gt, "has_gt": has_gt, "fname": fname}


def collate(items):
    """Items of one shape -> {'data': uint8 [N*H*W*4] (the N BGR frames, then the N masks), 'size': (N, H, W),
    'has_gt': bool [N], 'fname': [N]}.  One buffer, so pinning and the host-to-device copy are one transfer each."""
    h, w = items[0]["gt"].shape
    n = len(items)
    data = torch.empty(n * h * w * 4, dtype=torch.uint8)
    img, gt = views(data, n, h, w)
    for i, it in enumerate(items):
        if it["image"].shape != (h, w, 3) or it["gt"].shape != (h, w):
            raise ValueError("all frames of a batch must share a size")
        img[i] = torch.from_numpy(it["image"])
        gt[i] = torch.from_numpy(it["gt"])
    return {"data": data, "size": torch.tensor([n, h, w]), "has_gt": torch.tensor([bool(it["has_gt"]) for it in items]),
            "fname": [it["fname"] for it in items]}


def views(data, n, h, w):
    """The image [N,H,W,3] and mask [N,H,W] views of a collated buffer."""
    split = n * h * w * 3
    return data[:split].view(n, h, w, 3), data[split:split + n * h * w].view(n, h, w)


def pinned(data):
    """``data`` in page-locked memory, pinned in the calling thread.  Use this instead of a DataLoader's
    ``pin_memory=True``: the loader's pinning thread allocates page-locked memory at any moment, and such an allocation
    invalidates a CUDA graph the main thread is capturing (training steps and inference forwards are captured)."""
    return data if data.is_pinned() else data.pin_memory()


def upload(batch, device):
    """One host-to-device copy of a collated batch -> (image uint8 [N,H,W,3], gt uint8 [N,H,W], label stats)."""
    n, h, w = (int(v) for v in batch["size"])
    data = pinned(batch["data"]).to(device, non_blocking=True)
    img, gt = views(data, n, h, w)
    return img, gt, ops.label_stats_u8(gt)


def to_device(batch, device, augment=None, meanval=MEANVAL):
    """Collated batch -> {'image': f32 [N,3,H,W], 'gt': f32 [N,1,H,W]} on ``device``.

    augment None: the reference's make_img_gt_pair + ToTensor, bit for bit (ops.image_from_bgr8, ops.label_from_u8).
    Otherwise RandomHorizontalFlip + ScaleNRotate as the reference composes them, fused with the ingest
    (augment.affine_warp_u8): ``augment`` is a list of per-sample (flip, rot, scale) triples, or a random generator
    from which augment.draw_params draws them in the reference's order."""
    with torch.cuda.device(device):
        img, gt, stats = upload(batch, device)
        if augment is None:
            return {"image": ops.image_from_bgr8(img, meanval), "gt": ops.label_from_u8(gt, stats)}
        params = augment if isinstance(augment, (list, tuple)) else _augment.draw_params(int(img.shape[0]), rng=augment)
        return _augment.affine_warp_u8(img, gt, params, stats, meanval)
