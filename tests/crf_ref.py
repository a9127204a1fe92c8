"""Float64 numpy restatement of the dense CRF (csrc/crf.cu, DESIGN.md §29).

The lattice (scaling, elevation, the remainder-0 point, the rank, the barycentric weights and the packed keys) is
computed with the same unfused float64 operations in the same order as crf_elevate_kernel, so its keys and weights are
the kernel's bit for bit.  Everything after it (splat, blur, slice, the Gaussian, the softmax) is float64 here and fp32
on the device."""
import math

import numpy as np

D = 5
D1 = D + 1
Q_BITS = 10
Q_BIAS = 1 << (Q_BITS - 1)
KEY_BITS = D * Q_BITS + 3


def scales(theta_a, theta_b):
    """s_j = sqrt(2/3)·(d+1) / sqrt((j+1)(j+2)) / θ_j, θ = (θα, θα, θβ, θβ, θβ): the host's scale factors."""
    inv_std = math.sqrt(2.0 / 3.0) * D1
    theta = (theta_a,) * 2 + (theta_b,) * 3
    return [inv_std / math.sqrt(float((j + 1) * (j + 2))) / theta[j] for j in range(D)]


def elevate(frames, theta_a, theta_b):
    """frames uint8 [N,H,W,3] BGR -> (keys uint64 [P,6], weights float64 [P,6]): the 6 enclosing simplex vertices of
    every pixel's feature (x, y, R, G, B) and its barycentric weights, in crf_elevate_kernel's operation order."""
    n, h, w, _ = frames.shape
    s = scales(theta_a, theta_b)
    yy, xx = np.mgrid[0:h, 0:w]
    fr = frames.reshape(n, h, w, 3).astype(np.float64)
    v = [np.broadcast_to(xx, (n, h, w)).astype(np.float64).ravel(), np.broadcast_to(yy, (n, h, w)).astype(np.float64).ravel(),
         fr[..., 2].ravel(), fr[..., 1].ravel(), fr[..., 0].ravel()]
    p = n * h * w
    e = np.zeros((D1, p))
    sm = np.zeros(p)
    for j in range(D, 0, -1):
        cf = v[j - 1] * s[j - 1]
        e[j] = sm - float(j) * cf
        sm = sm + cf
    e[0] = sm
    down = 1.0 / D1
    t = e * down
    up, dn = np.ceil(t) * D1, np.floor(t) * D1
    rem0 = np.where(up - e < e - dn, up, dn).astype(np.int64)
    total = rem0.sum(0) // D1                      # an exact multiple: every rem0 is
    dif = e - rem0
    rank = np.zeros((D1, p), dtype=np.int64)
    for i in range(D):
        for j in range(i + 1, D1):
            less = dif[i] < dif[j]
            rank[i] += less
            rank[j] += ~less
    for i in range(D1):
        pos, neg = total > 0, total < 0
        c1 = pos & (rank[i] >= D1 - total)
        c2 = neg & (rank[i] < -total)
        rem0[i] = rem0[i] - D1 * c1 + D1 * c2
        rank[i] = np.where(c1, rank[i] + total - D1, np.where(c2, rank[i] + D1 + total, rank[i] + total))
    bary = np.zeros((D1 + 1, p))
    cols = np.arange(p)
    for i in range(D1):
        vi = (e[i] - rem0[i]) * down
        bary[D - rank[i], cols] += vi
        bary[D1 - rank[i], cols] -= vi
    bary[0] = bary[0] + (1.0 + bary[D1])
    frame = (np.arange(p) // (h * w)).astype(np.uint64)
    keys = np.zeros((p, D1), dtype=np.uint64)
    for r in range(D1):
        k = frame << np.uint64(KEY_BITS) | np.uint64(r << (D * Q_BITS))
        for i in range(D):
            key = rem0[i] + r - D1 * (rank[i] > D - r)
            q = (key - r) // D1
            assert np.all((key - r) % D1 == 0)
            assert np.all((q + Q_BIAS >= 0) & (q + Q_BIAS < 2 * Q_BIAS)), "key range"
            k = k | ((q + Q_BIAS).astype(np.uint64) << np.uint64(i * Q_BITS))
        keys[:, r] = k
    return keys, bary[:D1].T.copy()


def decode(keys):
    """Packed keys -> (frame, remainder class, the five coordinates)."""
    keys = keys.astype(np.uint64)
    frame = (keys >> np.uint64(KEY_BITS)).astype(np.int64)
    r = ((keys >> np.uint64(D * Q_BITS)) & np.uint64(7)).astype(np.int64)
    k = np.stack([D1 * (((keys >> np.uint64(i * Q_BITS)) & np.uint64(2 * Q_BIAS - 1)).astype(np.int64) - Q_BIAS) + r
                  for i in range(D)])
    return frame, r, k


def pack(frame, r, coords):
    q = (coords - r) // D1
    inside = np.all((q + Q_BIAS >= 0) & (q + Q_BIAS < 2 * Q_BIAS), axis=0)
    qc = np.clip(q + Q_BIAS, 0, 2 * Q_BIAS - 1).astype(np.uint64)
    k = frame.astype(np.uint64) << np.uint64(KEY_BITS) | (r.astype(np.uint64) << np.uint64(D * Q_BITS))
    for i in range(D):
        k = k | (qc[i] << np.uint64(i * Q_BITS))
    return k, inside


class Lattice:
    """One call's lattice: the sorted unique vertices, each entry's vertex, the 12 neighbours of every vertex."""

    def __init__(self, frames, theta_a, theta_b, weights_f32=False):
        self.keys, self.weights = elevate(frames, theta_a, theta_b)
        if weights_f32:                                # what the device stores
            self.weights = self.weights.astype(np.float32).astype(np.float64)
        self.pixels = self.keys.shape[0]
        self.uniq, inv = np.unique(self.keys.ravel(), return_inverse=True)
        self.vertex = inv.reshape(self.pixels, D1)
        self.m = self.uniq.size
        frame, r, k = decode(self.uniq)
        self.per_frame = np.bincount(frame, minlength=frames.shape[0])
        self.occupancy = np.bincount(inv, minlength=self.m)
        self.nbr = []
        for j in range(D1):
            pair = []
            for step in (-1, 1):
                c = k + step
                if j < D:
                    c[j] -= step * D1
                r2 = (r + step) % D1
                key, inside = pack(frame, r2, c)
                at = np.clip(np.searchsorted(self.uniq, key), 0, self.m - 1)
                pair.append(np.where(inside & (self.uniq[at] == key), at, -1))
            self.nbr.append(pair)

    def filter(self, values, reverse=False):
        """F: splat [P,C] onto the vertices, blur along the 6 directions with (1/4, 1/2, 1/4), slice.  ``reverse``
        blurs the directions in the opposite order: that filter is F's adjoint."""
        values = values.reshape(self.pixels, -1)
        c = values.shape[1]
        val = np.zeros((self.m, c))
        for ch in range(c):
            val[:, ch] = np.bincount(self.vertex.ravel(), weights=(self.weights * values[:, ch:ch + 1]).ravel(),
                                     minlength=self.m)
        for n1, n2 in (self.nbr[::-1] if reverse else self.nbr):
            pad = np.vstack([val, np.zeros((1, c))])     # index -1: absent, 0
            val = 0.5 * val + 0.25 * (pad[n1] + pad[n2])
        return np.einsum("pr,prc->pc", self.weights, val[self.vertex])


def gaussian_taps(theta_g):
    radius = int(math.ceil(3.0 * theta_g))
    d = np.arange(-radius, radius + 1, dtype=np.float64)
    return np.exp(-d * d / (2.0 * theta_g * theta_g))


def gaussian_filter(x, theta_g):
    """Correlation of [N,H,W] with the truncated separable Gaussian, pixels outside the frame absent (0)."""
    g = gaussian_taps(theta_g)
    radius = (g.size - 1) // 2
    n, h, w = x.shape
    out = np.zeros_like(x, dtype=np.float64)
    tmp = np.zeros_like(out)
    for dx in range(-radius, radius + 1):
        lo, hi = max(0, -dx), min(w, w - dx)
        if lo < hi:
            tmp[:, :, lo:hi] += g[dx + radius] * x[:, :, lo + dx:hi + dx]
    for dy in range(-radius, radius + 1):
        lo, hi = max(0, -dy), min(h, h - dy)
        if lo < hi:
            out[:, lo:hi, :] += g[dy + radius] * tmp[:, lo + dy:hi + dy, :]
    return out


def smoothness(q, theta_g):
    """S_l = (G * Q_l) / (G * 1), Q [L,N,H,W]."""
    ones = gaussian_filter(np.ones(q.shape[1:]), theta_g)
    return np.stack([gaussian_filter(ql, theta_g) / ones for ql in q])


def softmax(a):
    m = a.max(0, keepdims=True)
    e = np.exp(a - m)
    return e / e.sum(0, keepdims=True)


def mean_field_step(lat, a0, q, norm, w_a, w_g, theta_g):
    """One mean-field update: a = a⁰ + w_α B + w_γ S from the label probabilities q [K+1,N,H,W], with B = F(q) / F(1)
    (``norm`` = F(1) per pixel) and S the Gaussian message."""
    b = (lat.filter(q.reshape(q.shape[0], -1).T) / norm[:, None]).T.reshape(q.shape)
    s = smoothness(q, theta_g)
    return a0 + w_a * b + w_g * s


def dense_crf(frames, maps, iterations=5, w_a=10.0, theta_a=80.0, theta_b=13.0, w_g=3.0, theta_g=3.0, lattice=None,
              weights_f32=True):
    """frames uint8 [N,H,W,3], maps [K,N,H,W] -> refined maps float64 [K,N,H,W] (r_k = a_k - a_0 of the last
    iteration; the maps themselves for iterations == 0)."""
    z = np.asarray(maps, dtype=np.float64)
    if iterations == 0:
        return z.copy()
    if weights_f32:                                    # the device takes the weights as fp32
        w_a, w_g = float(np.float32(w_a)), float(np.float32(w_g))
    lat = Lattice(frames, theta_a, theta_b, weights_f32) if lattice is None else lattice
    k, n, h, w = z.shape
    a0 = np.concatenate([np.zeros((1, n, h, w)), z])
    q = softmax(a0)
    norm = lat.filter(np.ones((lat.pixels, 1)))[:, 0]
    for _ in range(iterations):
        a = mean_field_step(lat, a0, q, norm, w_a, w_g, theta_g)
        q = softmax(a)
    return a[1:] - a[0]
