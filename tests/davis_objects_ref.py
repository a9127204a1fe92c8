"""numpy restatement of the DAVIS-2017 per-object counts (DESIGN.md §24), the test oracle of
ops.davis_measures_objects and of ops.merge_objects.  Object k's masks are P = label == k and G = gt == k with the void
pixels (gt == 255) cleared from both; each pair is then scored by davis_measures_ref.counts unchanged."""
import numpy as np

import davis_measures_ref as M

VOID = 255


def object_counts(labels, gt, k_objects, r=None):
    """One frame: uint8 labels [H,W], uint8 annotation [H,W] -> [K][6] counts (object 1 first)."""
    labels, gt = np.asarray(labels), np.asarray(gt)
    void = gt == VOID
    out = []
    for k in range(1, k_objects + 1):
        p = (labels == k) & ~void
        g = (gt == k) & ~void
        out.append(M.counts(np.where(p, 1.0, -1.0).astype(np.float32), g.astype(np.uint8), r))
    return out


def merge(maps):
    """fp32 [K, ...] fused logits -> uint8 labels: 1 + the first k of the largest value where it is > 0, else 0."""
    maps = np.asarray(maps, np.float32)
    best = np.zeros(maps.shape[1:], np.float32)
    lab = np.zeros(maps.shape[1:], np.uint8)
    for k in range(maps.shape[0]):
        win = maps[k] > best                                   # NaN and ±0 compare False
        best = np.where(win, maps[k], best)
        lab = np.where(win, k + 1, lab).astype(np.uint8)
    return lab
