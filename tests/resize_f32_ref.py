"""A numpy restatement of Pillow's BILINEAR resize of an 'F' (fp32) image (libImaging/Resample.c, the 32bpc passes),
the arithmetic scipy 1.0's imresize(..., mode='F') ran; ops.resize_f32 is tested against it and it is tested against
PIL (tests/test_resize_f32.py).  Python floats and numpy float64 arrays are IEEE doubles evaluated one operation at a
time, with no fused multiply-add, as Pillow's C code is."""
import numpy as np


def coeffs(n_in, n_out):
    """[(xmin, [k...])] per output: precompute_coeffs' triangle weights, widened by the downscale factor and divided by
    their sum, in double (the 8-bit path rounds these to fixed point; the fp32 path does not)."""
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
        rows.append((xmin, ws))
    return rows


def _pass(x, rows, axis):
    """ss = 0.0; ss += (double)src * k per tap along ``axis`` (-2 = rows, -1 = columns) of x [..., H, W], stored as fp32."""
    xs = np.moveaxis(np.asarray(x, dtype=np.float32), axis, 0)
    ks = max(len(k) for _, k in rows)
    ss = np.zeros((len(rows),) + xs.shape[1:], dtype=np.float64)
    bcast = (-1,) + (1,) * (xs.ndim - 1)
    for t in range(ks):
        live = np.array([t < len(k) for _, k in rows])
        idx = np.array([min(xmin + t, xs.shape[0] - 1) for xmin, _ in rows])
        k = np.array([k[t] if t < len(k) else 0.0 for _, k in rows], dtype=np.float64)
        ss = np.where(live.reshape(bcast), ss + xs[idx].astype(np.float64) * k.reshape(bcast), ss)
    return np.moveaxis(ss.astype(np.float32), 0, axis)


def resize(arr, size):
    """fp32 [..., H, W] -> [..., h', w'] for size = (h', w'): each map as
    PIL.Image.fromarray(map, 'F').resize((w', h'), Image.BILINEAR)."""
    a = np.asarray(arr, dtype=np.float32)
    h, w = a.shape[-2:]
    oh, ow = size
    if (oh, ow) == (h, w):
        return a.copy()
    x, shift = a, 0
    vrows = coeffs(h, oh) if oh != h else None
    if ow != w:
        first, last = (vrows[0][0], vrows[-1][0] + len(vrows[-1][1])) if vrows else (0, h)
        x = _pass(x[..., first:last, :], coeffs(w, ow), -1)      # only the rows the vertical pass reads
        shift = first
    if vrows:
        x = _pass(x, [(xmin - shift, k) for xmin, k in vrows], -2)
    return x
