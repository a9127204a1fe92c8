"""DAVIS-2016 region (J) and boundary (F) scores from the device counts of ``ops.davis_measures`` (DESIGN.md §14).

The kernel produces six integers per frame; this module turns them into J and F (on the device, no synchronisation)
and a sequence's per-frame series into the benchmark's statistics: mean M, recall O and decay D.  As the DAVIS-2016
benchmark does, the statistics leave out a sequence's first frame (its annotation is the network's input) and its
last frame; the per-frame values of every frame are kept, so other conventions can be recomputed from them.
"""
import math

import numpy as np
import torch

BOUND_TH = 0.008                      # boundary tolerance as a fraction of the frame diagonal


def bound_pix(h, w):
    """Boundary tolerance radius in pixels: ceil(0.008 * sqrt(h² + w²)) (8 at 480x854, 18 at 1080x1920)."""
    return int(math.ceil(BOUND_TH * math.sqrt(h * h + w * w)))


def j_and_f(counts):
    """int [N,6] counts -> (J, F), float64 [N] each, on the counts' device.  J = |P∧G| / |P∨G| (1 when both masks are
    empty); F = 2PR / (P + R) of boundary precision P and recall R, with the benchmark's rules for empty boundaries."""
    c = counts.to(torch.float64)
    inter, union, n_fg, n_gt, fg_match, gt_match = c.unbind(-1)
    one, zero = torch.ones_like(inter), torch.zeros_like(inter)
    j = torch.where(union > 0, inter / union.clamp(min=1), one)
    # both boundaries empty: P = R = 1; only B(P) empty: P = 1, R = 0; only B(G) empty: P = 0, R = 1
    prec = torch.where(n_fg > 0, torch.where(n_gt > 0, fg_match / n_fg.clamp(min=1), zero), one)
    rec = torch.where(n_gt > 0, torch.where(n_fg > 0, gt_match / n_gt.clamp(min=1), zero), one)
    s = prec + rec
    f = torch.where(s > 0, 2 * prec * rec / torch.where(s > 0, s, one), zero)
    return j, f


def decay_bins(n):
    """The first indices of the benchmark's four decay bins of an n-frame series, plus the last index."""
    return (np.round(np.linspace(1, n, 5) + 1e-10) - 1).astype(int)


def statistics(values):
    """A sequence's per-frame series (every frame, first and last included) -> {'M', 'O', 'D'} over frames 1 .. n-2:
    M = mean, O = fraction above 0.5, D = mean of the first quarter bin minus mean of the last.  NaN when no frame
    is left."""
    x = np.asarray(values.cpu() if torch.is_tensor(values) else values, dtype=np.float64)[1:-1]
    if x.size == 0:
        return {"M": float("nan"), "O": float("nan"), "D": float("nan")}
    i = decay_bins(x.size)
    return {"M": float(np.mean(x)), "O": float(np.mean(x > 0.5)),
            "D": float(np.mean(x[i[0]:i[1] + 1]) - np.mean(x[i[3]:i[4] + 1]))}


class SequenceScores:
    """Accumulates device counts frame by frame without synchronising; ``result()`` reads them back once."""

    def __init__(self):
        self._counts = []

    def add(self, counts):
        self._counts.append(counts.reshape(-1, 6))

    def result(self):
        """{'J': per-frame list, 'F': per-frame list, 'counts': per-frame lists of six ints,
        'statistics': {'J': {M, O, D}, 'F': {M, O, D}}}."""
        if not self._counts:
            counts = torch.zeros((0, 6), dtype=torch.int32)
        else:
            counts = torch.cat([c.to(self._counts[0].device) for c in self._counts]).cpu()
        j, f = j_and_f(counts)
        return {"J": j.tolist(), "F": f.tolist(), "counts": counts.tolist(),
                "statistics": {"J": statistics(j), "F": statistics(f)}}
