"""numpy / scipy restatement of the DAVIS-2016 region (J) and boundary (F) measures and sequence statistics, written
from the definitions in DESIGN.md §14.  The test oracle of ops.davis_measures and osvos_pytorch_b200.evaluation."""
import math

import numpy as np
from scipy import ndimage


def bound_pix(h, w):
    return int(math.ceil(0.008 * math.hypot(h, w)))


def seg2bmap(seg):
    """Boundary map of a bool mask [H,W]."""
    seg = np.asarray(seg, dtype=bool)
    e = np.zeros_like(seg)
    s = np.zeros_like(seg)
    se = np.zeros_like(seg)
    e[:, :-1] = seg[:, 1:]
    s[:-1, :] = seg[1:, :]
    se[:-1, :-1] = seg[1:, 1:]
    b = (seg ^ e) | (seg ^ s) | (seg ^ se)
    b[-1, :] = seg[-1, :] ^ e[-1, :]
    b[:, -1] = seg[:, -1] ^ s[:, -1]
    b[-1, -1] = False
    return b


def disk(r):
    y, x = np.mgrid[-r:r + 1, -r:r + 1]
    return x * x + y * y <= r * r


def dilate(b, r):
    """Disk dilation with everything outside the frame background."""
    return ndimage.binary_dilation(b, structure=disk(r), border_value=0)


def counts(logit, gt_u8, r=None):
    """One frame: fp32 logits [H,W], uint8 annotation [H,W] -> the six integer counts of ops.davis_measures."""
    p = np.asarray(logit) > 0
    g = np.asarray(gt_u8) != 0
    r = bound_pix(*p.shape) if r is None else r
    bp, bg = seg2bmap(p), seg2bmap(g)
    return [int((p & g).sum()), int((p | g).sum()), int(bp.sum()), int(bg.sum()),
            int((bp & dilate(bg, r)).sum()), int((bg & dilate(bp, r)).sum())]


def j_and_f(c):
    inter, union, n_fg, n_gt, fg_match, gt_match = (float(v) for v in c)
    j = 1.0 if union == 0 else inter / union
    if n_fg == 0 and n_gt == 0:
        prec, rec = 1.0, 1.0
    elif n_fg == 0:
        prec, rec = 1.0, 0.0
    elif n_gt == 0:
        prec, rec = 0.0, 1.0
    else:
        prec, rec = fg_match / n_fg, gt_match / n_gt
    f = 0.0 if prec + rec == 0 else 2 * prec * rec / (prec + rec)
    return j, f


def statistics(series):
    """Per-frame series of a whole sequence -> (M, O, D) over frames 1 .. n-2; NaN when none is left."""
    x = np.asarray(series, dtype=np.float64)[1:-1]
    if x.size == 0:
        return float("nan"), float("nan"), float("nan")
    ids = np.round(np.linspace(1, x.size, 5) + 1e-10).astype(int) - 1
    bins = [x[ids[i]:ids[i + 1] + 1] for i in range(4)]
    return float(np.mean(x)), float(np.mean(x > 0.5)), float(np.mean(bins[0]) - np.mean(bins[3]))
