"""Seeded BGR frames for the JPEG encoder's tests: the size matrix, the qualities and five kinds of content."""
import numpy as np

SIZES = [(1, 1), (1, 17), (7, 9), (8, 8), (16, 16), (17, 33), (97, 131), (240, 427), (480, 854)]
QUALITIES = [1, 5, 50, 75, 95, 100]
KINDS = ["noise", "smooth", "flat", "saturated", "overlay"]


def frame(h, w, kind, seed=0):
    """uint8 [h][w][3] BGR."""
    rng = np.random.default_rng([h, w, KINDS.index(kind), seed])
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "smooth":
        ph = rng.random(3) * 6.28
        return np.stack([128 + 100 * np.sin(xx / 17.0 + ph[c]) * np.cos(yy / 23.0 - ph[c]) for c in range(3)],
                        -1).astype(np.uint8)
    if kind == "flat":
        return np.broadcast_to(rng.integers(0, 256, 3, dtype=np.uint8), (h, w, 3)).copy()
    if kind == "saturated":                                        # hard 0 / 255 edges in every channel
        return (((xx[..., None] // 3 + yy[..., None] // 5 + np.arange(3)) % 2) * 255).astype(np.uint8)
    # a smooth picture with a blended blob and its black outline, as ops.overlay_mask draws them
    base = frame(h, w, "smooth", seed).astype(np.int64)
    blob = (yy - 0.5 * h) ** 2 / max(0.3 * h, 1) ** 2 + (xx - 0.45 * w) ** 2 / max(0.3 * w, 1) ** 2 < 1
    inner = np.zeros_like(blob)
    inner[1:-1, 1:-1] = blob[1:-1, 1:-1] & blob[:-2, 1:-1] & blob[2:, 1:-1] & blob[1:-1, :-2] & blob[1:-1, 2:]
    out = base.copy()
    out[blob] = (base[blob] + np.array([0, 0, 255]) + 1) >> 1
    out[blob & ~inner] = 0
    return out.astype(np.uint8)


def random_shapes(count, seed=7, hmax=300, wmax=300):
    rng = np.random.default_rng(seed)
    return [(int(rng.integers(1, hmax)), int(rng.integers(1, wmax))) for _ in range(count)]
