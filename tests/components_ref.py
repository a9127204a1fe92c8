"""numpy / scipy restatement of ops.connected_components and ops.filter_components (DESIGN.md §30).

Labels are scipy.ndimage.label's; squared distances are integers, formed from the indices of the nearest feature that
scipy's exact Euclidean distance transform returns (adaptation_ref.squared_distance_to), so no float enters a
comparison."""
import numpy as np
from scipy import ndimage

from adaptation_ref import squared_distance_to

STRUCTURES = {4: ndimage.generate_binary_structure(2, 1), 8: np.ones((3, 3), bool)}


def label(mask, connectivity=8):
    """One frame: (labels int32 [H,W], count)."""
    lab, n = ndimage.label(np.asarray(mask) != 0, STRUCTURES[connectivity])
    return lab.astype(np.int32), int(n)


def connected_components(masks, connectivity=8):
    """[N,H,W] -> (labels int32 [N,H,W], counts int32 [N])."""
    out = [label(m, connectivity) for m in masks]
    return np.stack([o[0] for o in out]), np.array([o[1] for o in out], np.int32)


def largest(lab, n):
    """The label of the component with the most pixels, ties to the smallest label; 0 when there is none."""
    if n == 0:
        return 0
    areas = np.bincount(lab.ravel(), minlength=n + 1)[1:]
    return int(np.argmax(areas)) + 1                 # argmax takes the first of equal maxima


def filter_frame(z, prior, mode, radius, connectivity):
    """One object, one frame: z fp32 [H,W], prior bool [H,W] or None -> (z' fp32, kept bool, stats [4])."""
    z = np.asarray(z, np.float32)
    f = z > 0
    lab, n = label(f, connectivity)
    keep_labels = {largest(lab, n)} if n else set()
    if mode == "near" and n and prior is not None and prior.any():
        d = squared_distance_to(prior)
        mind = np.full(n + 1, np.iinfo(np.int64).max, np.int64)
        np.minimum.at(mind, lab[f], d[f])
        near = {i for i in range(1, n + 1) if mind[i] <= radius * radius}
        if near:
            keep_labels = near
    kept = f & np.isin(lab, sorted(keep_labels))
    dropped = f & ~kept
    out = z.copy()
    out[dropped] = -z[dropped]
    return out, kept, np.array([n, len(keep_labels), int(f.sum()), int(dropped.sum())], np.int32)


def filter_components(maps, mode, radius=32, connectivity=8, prior=None):
    """maps fp32 [K,N,H,W], prior uint8 [K,H,W] or None -> (out fp32 [K,N,H,W], kept uint8 [K,N,H,W], stats [K,N,4]).
    "near" takes the frames in order: frame j > 0 is measured against frame j - 1's kept mask."""
    maps = np.asarray(maps, np.float32)
    k, n = maps.shape[:2]
    out, kept, stats = np.empty_like(maps), np.zeros(maps.shape, np.uint8), np.zeros((k, n, 4), np.int32)
    for o in range(k):
        p = None if prior is None else np.asarray(prior[o]) != 0
        for j in range(n):
            out[o, j], kk, stats[o, j] = filter_frame(maps[o, j], p, mode, radius, connectivity)
            kept[o, j] = kk
            p = kk
    return out, kept, stats
