"""Maps for the PNG encoder tests (tests/test_png.py, tests/test_gpu_png.py), all seeded."""
import numpy as np

# row widths around the segment split (png_ref.SEGMENT_BYTES // (w + 1) rows per segment)
SHAPES = [(1, 1), (1, 57), (33, 1), (7, 9), (40, 56), (97, 131), (240, 427), (480, 854), (3, 16383), (2, 16384),
          (5, 8191), (4, 8192)]


def smooth_field(h, w, seed):
    from scipy.ndimage import gaussian_filter
    z = gaussian_filter(np.random.default_rng(seed).standard_normal((h, w)), sigma=max(1.0, h / 24))
    return z / max(z.std(), 1e-12)


def bytescale(h, w, seed=0):
    """A sigmoid map bytescaled as scipy.misc.imsave does: steep, so about three quarters of the bytes are 0 or 255, as
    in the network's test-time maps."""
    from scipy.special import expit
    p = expit(20 * smooth_field(h, w, seed))
    lo, hi = p.min(), p.max()
    return np.round(255 * (p - lo) / max(hi - lo, 1e-12)).astype(np.uint8)


def mask(h, w, seed=0):
    return np.where(smooth_field(h, w, seed) > 0, 255, 0).astype(np.uint8)


def noise(h, w, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (h, w), dtype=np.uint8)


def fibonacci(seed=0):
    """One row whose Sub-filtered bytes have Fibonacci-like counts and no run longer than 3: with the end-of-block code
    (count 1) and the filter type byte (a 1), the literal counts are 1, 1, 2, 3, 5, ..., 1597, so the filter picks Sub
    and an unlimited Huffman code for the row is 16 bits deep."""
    fib = [1, 2]
    while len(fib) < 16:
        fib.append(fib[-1] + fib[-2])
    counts = fib[::-1]                       # value 0 the most frequent
    counts[1] -= 1                           # the type byte of Sub is a 1
    vals = np.repeat(np.arange(16), counts)
    rng = np.random.default_rng(seed)
    rng.shuffle(vals)
    for _ in range(100):                     # break runs of 4: swap the 4th byte with a random one
        bad = np.flatnonzero((vals[3:] == vals[2:-1]) & (vals[2:-1] == vals[1:-2]) & (vals[1:-2] == vals[:-3])) + 3
        if not len(bad):
            break
        for i in bad:
            j = rng.integers(len(vals))
            vals[i], vals[j] = vals[j], vals[i]
    return (np.cumsum(vals) & 255)[None].astype(np.uint8)             # Sub undoes the running sum


def content(kind, h, w, seed=0):
    if kind == "zeros":
        return np.zeros((h, w), np.uint8)
    if kind == "ones":
        return np.full((h, w), 255, np.uint8)
    return {"bytescale": bytescale, "mask": mask, "noise": noise}[kind](h, w, seed)


KINDS = ["zeros", "ones", "mask", "bytescale", "noise"]
