"""Rebuilds the DAVIS-layout tree stored in tests/golden/reference_davis.npz (made by make_golden_davis.py)."""
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_davis.npz")


def load():
    with np.load(PATH, allow_pickle=False) as z:
        return {k: z[k] for k in z.files}


def write_tree(fx, root):
    """Writes the fixture's encoded files under ``root``; returns ``root``."""
    for key, data in fx.items():
        if key.startswith("file:"):
            path = os.path.join(root, key[len("file:"):])
            os.makedirs(os.path.dirname(path), exist_ok=True)
            data.tofile(path)
    return str(root)


def pair(fx, img_rel, has_gt=True):
    key = img_rel + ("" if has_gt else ":nolabel")
    return fx[f"pair.{key}.image"], fx[f"pair.{key}.gt"]
