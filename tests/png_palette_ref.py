"""Restatement of the palette PNG files (DESIGN.md §24): the encoder's palette file is png_ref.encode's grayscale file
with IHDR colour type 3 and a PLTE chunk after IHDR; the decoder turns 1/2/4/8-bit palette rows into raw indices."""
import io
import struct
import zlib

import numpy as np

import png_ref as P


def encode(a, palette):
    """uint8 [H,W] indices and PLTE bytes -> the palette PNG file the kernels write."""
    gray = P.encode(a)
    cs = P.chunks(gray)
    w, h = struct.unpack(">II", cs[0][1][:8])
    ihdr = P.chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 3, 0, 0, 0))
    head = len(P.SIGNATURE) + 25
    return P.SIGNATURE + ihdr + P.chunk(b"PLTE", bytes(palette)) + gray[head:]


def strip_palette(data):
    """A palette file -> the grayscale file of the same indices: IHDR colour type 0, the PLTE chunk dropped."""
    cs = P.chunks(data)
    out = [P.SIGNATURE]
    for kind, payload, _ in cs:
        if kind == b"PLTE":
            continue
        if kind == b"IHDR":
            payload = payload[:9] + b"\x00" + payload[10:]
        out.append(P.chunk(kind, payload))
    return b"".join(out)


def _unfilter(raw, h, rb):
    rows = np.frombuffer(raw, np.uint8).reshape(h, rb + 1)
    out = np.zeros((h, rb), np.int32)
    prior = np.zeros(rb, np.int32)
    for y in range(h):
        t, f = int(rows[y, 0]), rows[y, 1:].astype(np.int32)
        cur = np.zeros(rb, np.int32)
        for x in range(rb):                                    # one byte per "pixel" (bpp 1 for depths <= 8)
            a = cur[x - 1] if x else 0
            b = prior[x]
            c = prior[x - 1] if x else 0
            pred = [0, a, b, (a + b) // 2, int(P._paeth(np.int32(a), np.int32(b), np.int32(c)))][t]
            cur[x] = (f[x] + pred) & 255
        out[y] = cur
        prior = cur
    return out.astype(np.uint8)


def decode_index(data):
    """A non-interlaced palette PNG (depth 1, 2, 4 or 8) -> (uint8 [H,W] raw indices, PLTE bytes)."""
    cs = P.chunks(data)
    w, h, depth, ctype, _, _, inter = struct.unpack(">IIBBBBB", cs[0][1])
    assert ctype == 3 and inter == 0 and depth in (1, 2, 4, 8)
    raw = zlib.decompress(b"".join(p for k, p, _ in cs if k == b"IDAT"))
    rb = (w * depth + 7) // 8
    rows = _unfilter(raw, h, rb)
    per = 8 // depth
    x = np.arange(w)
    shift = 8 - depth * (x % per + 1)
    out = (rows[:, x // per] >> shift) & ((1 << depth) - 1)
    plte = next(p for k, p, _ in cs if k == b"PLTE")
    return out.astype(np.uint8), plte


def davis_palette(n):
    """The first n entries of the DAVIS palette: object k's colour from the bits of k (the toolkit's colour map)."""
    out = []
    for k in range(n):
        r = g = b = 0
        c = k
        for j in range(8):
            r |= ((c >> 0) & 1) << (7 - j)
            g |= ((c >> 1) & 1) << (7 - j)
            b |= ((c >> 2) & 1) << (7 - j)
            c >>= 3
        out += [r, g, b]
    return bytes(out)


def pillow_palette_png(idx, entries, transparency=None):
    """uint8 [H,W] indices -> the palette PNG Pillow writes (depth 1/2/4/8 from the palette length)."""
    from PIL import Image
    im = Image.fromarray(idx, "P")
    im.putpalette(davis_palette(entries))
    buf = io.BytesIO()
    im.save(buf, "PNG", **({} if transparency is None else {"transparency": transparency}))
    return buf.getvalue()
