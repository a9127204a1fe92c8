"""Training-time augmentation on the device (SURVEY.md 8f item 2): the reference's ``RandomHorizontalFlip`` followed
by ``ScaleNRotate(rots=(-30, 30), scales=(.75, 1.25))`` (dataloaders/custom_transforms.py:7-54, :87-100; composed at
train_online.py:92-94 and train_parent.py:108-110), applied to a GPU-resident batch by one gather kernel per tensor
instead of cv2 on a DataLoader worker.  The random draws use Python's ``random`` in the reference's order (flip
first, then rotation, then scale) so a seeded run picks the same transformations.  Matrices follow OpenCV's
``getRotationMatrix2D`` / ``warpAffine`` (inverse map); the arithmetic is in csrc/augment.cu.
"""
import ctypes
import math
import random

import torch

from . import _native as nat
from . import ops


def rotation_matrix(center, angle_deg, scale):
    """cv2.getRotationMatrix2D: [[a, b, (1-a)cx - b cy], [-b, a, b cx + (1-a) cy]], a = s cos, b = s sin."""
    a = scale * math.cos(math.radians(angle_deg))
    b = scale * math.sin(math.radians(angle_deg))
    cx, cy = center
    return [a, b, (1.0 - a) * cx - b * cy, -b, a, b * cx + (1.0 - a) * cy]


def invert_affine(m):
    """The dst->src matrix cv::warpAffine derives from M (no WARP_INVERSE_MAP)."""
    m = list(m)
    d = m[0] * m[4] - m[1] * m[3]
    d = 1.0 / d if d != 0 else 0.0
    a11, a22 = m[4] * d, m[0] * d
    m[0], m[1], m[3], m[4] = a11, m[1] * -d, m[3] * -d, a22
    b1 = -m[0] * m[2] - m[1] * m[5]
    b2 = -m[3] * m[2] - m[4] * m[5]
    m[2], m[5] = b1, b2
    return m


def draw_params(n, rots=(-30, 30), scales=(.75, 1.25), rng=random):
    """Per-sample (flip, rot, scale) drawn like the reference's transforms: RandomHorizontalFlip.__call__ draws
    first (custom_transforms.py:92), then ScaleNRotate draws rot and sc (:25-29)."""
    out = []
    for _ in range(n):
        flip = rng.random() < 0.5
        rot = (rots[1] - rots[0]) * rng.random() - (rots[1] - rots[0]) / 2
        sc = (scales[1] - scales[0]) * rng.random() - (scales[1] - scales[0]) / 2 + 1
        out.append((flip, rot, sc))
    return out


def _warp_tables(params, n, h, w):
    """Host tables of osvos_affine_warp*: n inverted 2x3 matrices and n flip flags."""
    if len(params) != n:
        raise ValueError("one (flip, rot, scale) triple per sample")
    mats = (ctypes.c_double * (6 * n))()
    flips = (ctypes.c_int * n)()
    for i, (flip, rot, sc) in enumerate(params):
        inv = invert_affine(rotation_matrix((w / 2, h / 2), rot, sc))
        mats[6 * i:6 * i + 6] = inv
        flips[i] = int(bool(flip))
    return mats, flips


def affine_warp(x, params, mode):
    """x [n,c,h,w] fp32 CUDA -> warped copy.  params: list of n (flip, rot_degrees, scale); mode 'cubic'|'nearest'."""
    lib = nat.load()
    ops._require_cuda(x, "x")
    x = x.contiguous().float()
    n, c, h, w = (int(v) for v in x.shape)
    mats, flips = _warp_tables(params, n, h, w)
    out = torch.empty_like(x)
    ops._count((n + 31) // 32)
    with torch.cuda.device(x.device):
        nat.check(lib.osvos_affine_warp(x.data_ptr(), out.data_ptr(), mats, flips, n, c, h, w,
                                        0 if mode == "cubic" else 1, torch.cuda.current_stream().cuda_stream),
                  "osvos_affine_warp")
    return out


def augment_batch(sample, rots=(-30, 30), scales=(.75, 1.25), rng=random, params=None):
    """{'image': [n,3,h,w], 'gt': [n,1,h,w]} on the GPU -> augmented copy (image bicubic, gt nearest: DAVIS masks are
    0/1 after ``gt / gt.max()``, the case in which the reference selects INTER_NEAREST, custom_transforms.py:45-48)."""
    n = int(sample["image"].shape[0])
    params = draw_params(n, rots, scales, rng) if params is None else params
    return {"image": affine_warp(sample["image"], params, "cubic"), "gt": affine_warp(sample["gt"], params, "nearest")}


def affine_warp_u8(image_u8, gt_u8, params, stats=None, meanval=ops.MEANVAL, index=None, ids=False):
    """RandomHorizontalFlip + ScaleNRotate straight from decoded bytes: image_u8 uint8 [n,h,w,3] BGR and gt_u8 uint8
    [n,h,w] on the GPU -> {'image': f32 [n,3,h,w], 'gt': f32 [n,1,h,w]}, bit-identical to ingesting them
    (ops.image_from_bgr8 / ops.label_from_u8) and then warping with affine_warp.  The image is warped bicubic; each mask
    nearest if it is binary and bicubic otherwise, the reference's per-sample rule (custom_transforms.py:46-49), decided
    on the device from ``stats`` (ops.label_stats_u8, computed here when None).

    ``index``: a sequence of frame indices.  Then image_u8, gt_u8 and stats are stores of any number of frames, and the
    output has len(index) samples, sample i warped from frame index[i] (repeats allowed): the same result as gathering
    those frames into a contiguous batch first, without the copy.  ``stats`` is required in this mode (computing it over
    a whole store per batch would cost more than the warp); an index outside the store raises IndexError.

    ``ids``: False or None (gt_u8 holds masks) or "all" / k (1..254): gt_u8 holds DAVIS-2017 object-id maps, and the gt is their
    label (ops.labels_from_ids with object None / k: 1 object, 0 background, -1 void), always sampled nearest
    (osvos_affine_warp_ids); ``stats`` is then unused."""
    lib = nat.load()
    obj = None if ids is None or ids is False else ops._id_object(ids)
    img = ops._require_u8(image_u8, "image_u8", 4)
    gt = ops._require_u8(gt_u8, "gt_u8", 3)
    n, h, w, c = (int(v) for v in img.shape)
    if c != 3 or tuple(gt.shape) != (n, h, w):
        raise ValueError("image_u8 must be [n,h,w,3] and gt_u8 [n,h,w]")
    m = n if index is None else len(index)
    mats, flips = _warp_tables(params, m, h, w)
    if obj is not None:
        stats = None
    if index is None:
        stats = ops.label_stats_u8(gt) if stats is None and obj is None else stats
    else:
        if stats is None and obj is None:
            raise ValueError("affine_warp_u8(index=...) needs the store's label stats (ops.label_stats_u8)")
        if stats is not None and tuple(stats.shape) != (n, 2):
            raise ValueError(f"stats must be [{n},2] for a store of {n} frames, got {tuple(stats.shape)}")
        idx = [int(i) for i in index]
        bad = [i for i in idx if not 0 <= i < n]
        if bad:
            raise IndexError(f"frame indices {bad[:8]} outside a store of {n} frames")
        idx = (ctypes.c_int * m)(*idx)
    out_i = torch.empty((m, 3, h, w), dtype=torch.float32, device=img.device)
    out_g = torch.empty((m, 1, h, w), dtype=torch.float32, device=img.device)
    ops._count(2 * ((m + 31) // 32))
    with torch.cuda.device(img.device):
        if obj is not None:
            stream = torch.cuda.current_stream().cuda_stream
            if index is None:
                nat.check(lib.osvos_affine_warp_u8(img.data_ptr(), None, None, out_i.data_ptr(), None, mats, flips, n,
                                                   h, w, *(float(v) for v in meanval), stream), "osvos_affine_warp_u8")
            else:
                nat.check(lib.osvos_affine_warp_u8_indexed(img.data_ptr(), None, None, out_i.data_ptr(), None, idx, mats,
                                                           flips, m, n, h, w, *(float(v) for v in meanval), stream),
                          "osvos_affine_warp_u8_indexed")
            nat.check(lib.osvos_affine_warp_ids(gt.data_ptr(), out_g.data_ptr(), None if index is None else idx, mats,
                                                flips, m, n, h, w, obj, stream), "osvos_affine_warp_ids")
        elif index is None:
            nat.check(lib.osvos_affine_warp_u8(img.data_ptr(), gt.data_ptr(), stats.data_ptr(), out_i.data_ptr(),
                                               out_g.data_ptr(), mats, flips, n, h, w, *(float(v) for v in meanval),
                                               torch.cuda.current_stream().cuda_stream), "osvos_affine_warp_u8")
        else:
            nat.check(lib.osvos_affine_warp_u8_indexed(img.data_ptr(), gt.data_ptr(), stats.data_ptr(),
                                                       out_i.data_ptr(), out_g.data_ptr(), idx, mats, flips, m, n, h, w,
                                                       *(float(v) for v in meanval),
                                                       torch.cuda.current_stream().cuda_stream),
                      "osvos_affine_warp_u8_indexed")
    return {"image": out_i, "gt": out_g}
