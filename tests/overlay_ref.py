"""numpy restatement of ops.overlay_mask (csrc/jpeg_encode.cu, DESIGN.md §23): the rule that replaces the reference's
dataloaders/helpers.py overlay_mask (a float blend and cv2.findContours + cv2.drawContours)."""
import numpy as np


def edge(fg):
    """bool [..., H, W] -> foreground pixels with a 4-neighbour in the background or outside the frame."""
    p = np.pad(fg, [(0, 0)] * (fg.ndim - 2) + [(1, 1), (1, 1)])
    inner = p[..., :-2, 1:-1] & p[..., 2:, 1:-1] & p[..., 1:-1, :-2] & p[..., 1:-1, 2:]
    return fg & ~inner


def overlay(frames, logits, color=(0, 0, 255)):
    """uint8 [N,H,W,3] BGR and fp32 logits [N,1,H,W] / [N,H,W] -> uint8 [N,H,W,3]."""
    v = np.asarray(frames).astype(np.int64)
    fg = np.asarray(logits, np.float32).reshape(v.shape[:-1]) > 0            # NaN and +-0 are background
    e = edge(fg)
    out = np.where(fg[..., None], (v + np.asarray(color, np.int64) + 1) >> 1, v)
    out[e] = 0
    return out.astype(np.uint8)
