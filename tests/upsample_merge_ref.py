"""numpy restatement of ops.upsample_merge_objects (DESIGN.md §27): every object's fused map resized as Pillow's 'F'
BILINEAR resize (tests/resize_f32_ref.py), then merged (tests/davis_objects_ref.py)."""
import numpy as np

import davis_objects_ref
import resize_f32_ref


def upsample_merge(maps, size):
    """fp32 [K, ..., h, w] -> uint8 labels [..., h', w'] for size = (h', w')."""
    maps = np.asarray(maps, np.float32)
    return davis_objects_ref.merge(np.stack([resize_f32_ref.resize(m, size) for m in maps]))
