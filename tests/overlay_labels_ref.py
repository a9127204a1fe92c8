"""numpy restatement of ops.overlay_labels (csrc/jpeg_encode.cu, DESIGN.md §25): the overlay of tests/overlay_ref.py
for a label map of K objects, each in its palette colour with its own outline."""
import numpy as np


def edge(labels):
    """uint8 [..., H, W] -> pixels of an object (id != 0) with a 4-neighbour of another id or outside the frame."""
    lab = np.asarray(labels).astype(np.int32)
    p = np.pad(lab, [(0, 0)] * (lab.ndim - 2) + [(1, 1), (1, 1)], constant_values=-1)
    inner = ((p[..., :-2, 1:-1] == lab) & (p[..., 2:, 1:-1] == lab) & (p[..., 1:-1, :-2] == lab)
             & (p[..., 1:-1, 2:] == lab))
    return (lab != 0) & ~inner


def overlay(frames, labels, palette):
    """uint8 [N,H,W,3] BGR, uint8 labels [N,H,W] and PLTE bytes (RGB triples) -> uint8 [N,H,W,3]: id 0 keeps the
    frame, an object's edge is black, the rest of object k is (v + c_k + 1) >> 1 with c_k entry k in BGR order
    ((0, 0, 0) past the palette's end)."""
    v = np.asarray(frames).astype(np.int64)
    lab = np.asarray(labels).reshape(v.shape[:-1])
    rgb = np.frombuffer(bytes(palette), np.uint8).reshape(-1, 3)
    table = np.zeros((256, 3), np.int64)
    table[:len(rgb)] = rgb[:, ::-1]
    out = np.where((lab != 0)[..., None], (v + table[lab] + 1) >> 1, v)
    out[edge(lab)] = 0
    return out.astype(np.uint8)
