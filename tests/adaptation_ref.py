"""numpy / scipy restatement of the online adaptation targets (ops.adaptation_labels, DESIGN.md §28).

Squared distances are integers: scipy's exact Euclidean distance transform is asked for the indices of the nearest
feature, and the squared distance is formed from them as (i - ii)² + (j - jj)², so no float enters a comparison."""
import math

import numpy as np
from scipy import ndimage


def threshold(alpha):
    """float32(ln(alpha / (1 - alpha))), computed in float64."""
    return np.float32(math.log(alpha / (1.0 - alpha)))


def squared_distance_to(features):
    """int64 [H,W]: min over feature pixels q of |p - q|²; None when there is no feature."""
    features = np.asarray(features, dtype=bool)
    if not features.any():
        return None
    _, (ii, jj) = ndimage.distance_transform_edt(~features, return_indices=True)
    i, j = np.indices(features.shape)
    return (i - ii).astype(np.int64) ** 2 + (j - jj).astype(np.int64) ** 2


def eroded(mask, e):
    """E: the pixels of M whose squared distance to every background pixel inside the frame exceeds e²."""
    m = np.asarray(mask) != 0
    d_bg = squared_distance_to(~m)
    if d_bg is None:                                    # no background: nothing erodes the mask
        return m
    return m & (d_bg > e * e)


def frame_labels(logits, mask, alpha, e, d):
    """One frame: logits fp32 [H,W], mask uint8 [H,W] -> (labels fp32 [H,W], counts int32 [3])."""
    e_set = eroded(mask, e)
    dist = squared_distance_to(e_set)
    negative = np.zeros(e_set.shape, dtype=bool) if dist is None else dist > d * d
    positive = ~negative & (np.asarray(logits, dtype=np.float32) > threshold(alpha))
    labels = np.full(e_set.shape, -1.0, dtype=np.float32)
    labels[negative] = 0.0
    labels[positive] = 1.0
    return labels, np.array([e_set.sum(), positive.sum(), negative.sum()], dtype=np.int32)


def adaptation_labels(logits, masks, alpha, e, d):
    """Batch form: logits [N,1,H,W] fp32, masks [N,H,W] uint8 -> (labels [N,1,H,W] fp32, counts [N,3] int32)."""
    out = [frame_labels(logits[k, 0], masks[k], alpha, e, d) for k in range(masks.shape[0])]
    return np.stack([o[0] for o in out])[:, None], np.stack([o[1] for o in out])
