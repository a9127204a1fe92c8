"""A numpy restatement of Pillow's 8-bit Image.resize (libImaging/Resample.c and Geometry.c ImagingScaleAffine), the
arithmetic scipy 1.0's imresize ran for uint8 input; ops.resize_u8 is tested against it and it is tested against PIL
(tests/test_resize.py).  Python floats are IEEE doubles evaluated one operation at a time, as Pillow's C code is."""
import numpy as np

PRECISION_BITS = 22


def bilinear_tables(n_in, n_out):
    """[(xmin, [k...])] per output: the triangle filter widened by the downscale factor, normalised, 22-bit fixed point."""
    scale = n_in / n_out
    fs = max(scale, 1.0)
    support = fs * 1.0
    ss = 1.0 / fs
    rows = []
    for o in range(n_out):
        center = (o + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), n_in)
        ws = []
        ww = 0.0
        for x in range(xmax - xmin):
            t = abs((x + xmin - center + 0.5) * ss)
            w = 1.0 - t if t < 1.0 else 0.0
            ws.append(w)
            ww += w
        if ww != 0.0:
            ws = [w / ww for w in ws]
        rows.append((xmin, [int(w * (1 << PRECISION_BITS) - 0.5) if w < 0 else int(w * (1 << PRECISION_BITS) + 0.5)
                            for w in ws]))
    return rows


def _taps(rows, n_in):
    """Source indices and weights [out, ksize], zero weights past each output's own count."""
    ks = max(len(k) for _, k in rows)
    idx = np.zeros((len(rows), ks), dtype=np.int64)
    wts = np.zeros((len(rows), ks), dtype=np.int64)
    for o, (xmin, k) in enumerate(rows):
        idx[o] = np.minimum(xmin + np.arange(ks), n_in - 1)
        wts[o, :len(k)] = k
    return idx, wts


def _pass(x, rows, axis):
    """2^21 + sum over taps of src * k along ``axis`` (0 = rows, 1 = columns) of x [H,W,C], clipped to 8 bits."""
    idx, wts = _taps(rows, x.shape[axis])
    acc = np.full((len(rows),) + tuple(np.delete(x.shape, axis)), 1 << (PRECISION_BITS - 1), dtype=np.int64)
    xs = np.moveaxis(x, axis, 0)
    for t in range(idx.shape[1]):
        acc += xs[idx[:, t]] * wts[:, t].reshape((-1,) + (1,) * (xs.ndim - 1))
    return np.moveaxis(_clip8(acc), 0, axis).astype(np.int64)


def _clip8(acc):
    return np.where(acc <= 0, 0, np.where(acc >= 1 << (PRECISION_BITS + 8), 255, acc >> PRECISION_BITS)).astype(np.uint8)


def nearest_index(n_in, n_out):
    """ImagingScaleAffine's running sum: xo = scale / 2, then xo += scale per output."""
    scale = n_in / n_out
    xo = scale * 0.5
    idx = []
    for _ in range(n_out):
        idx.append(min(int(xo), n_in - 1))
        xo += scale
    return np.array(idx, dtype=np.int64)


def resize(arr, size, mode="bilinear"):
    """uint8 [H,W] or [H,W,C] -> [h', w'(, C)] for size = (h', w'), as PIL.Image.fromarray(arr).resize((w', h'))."""
    a = np.asarray(arr, dtype=np.uint8)
    h, w = a.shape[:2]
    oh, ow = size
    if (oh, ow) == (h, w):
        return a.copy()
    if mode == "nearest":
        return a[nearest_index(h, oh)][:, nearest_index(w, ow)]
    x = a.reshape(h, w, -1).astype(np.int64)
    if ow != w:
        vrows = bilinear_tables(h, oh) if oh != h else None
        first, last = (vrows[0][0], vrows[-1][0] + len(vrows[-1][1])) if vrows else (0, h)
        x = _pass(x[first:last], bilinear_tables(w, ow), 1)
        shift = first
    else:
        shift = 0
    if oh != h:
        rows = [(xmin - shift, ks) for xmin, ks in bilinear_tables(h, oh)]
        x = _pass(x, rows, 0)
    return x.astype(np.uint8).reshape((oh, ow) + a.shape[2:])
