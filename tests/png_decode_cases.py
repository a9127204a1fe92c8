"""PNG files for the decoder tests (tests/test_png_decode.py, tests/test_gpu_png_decode.py): the same maps written by
Pillow, cv2 and the project's own format (tests/png_ref.py), hand-built files with true and false cuts, files outside
the device subset, and corrupt streams with valid chunk CRCs.  All seeded."""
import io
import struct
import zlib

import numpy as np

import png_cases as C
import png_ref as P

SIGNATURE = b"\x89PNG\r\n\x1a\n"
FLUSH = b"\x00\x00\xff\xff"
SHAPES = C.SHAPES + [(1, 9), (9, 1), (5, 13), (17, 23)]
SMALL = [s for s in SHAPES if s[0] * s[1] <= 6000]


def chunk(kind, body):
    return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", zlib.crc32(kind + body))


def build(h, w, idats, depth=8, colour=0, interlace=0, extra=()):
    """A PNG file from IDAT payloads; ``extra``: (kind, body) chunks between IHDR and the first IDAT."""
    out = SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, colour, 0, 0, interlace))
    for kind, body in extra:
        out += chunk(kind, body)
    for body in idats:
        out += chunk(b"IDAT", body)
    return out + chunk(b"IEND", b"")


def chunks(data):
    """[(kind, body)] of a PNG file."""
    out, p = [], 8
    while p < len(data):
        ln, = struct.unpack(">I", data[p:p + 4])
        out.append((data[p + 4:p + 8], data[p + 8:p + 8 + ln]))
        p += 12 + ln
    return out


def stream_of(data):
    return b"".join(body for kind, body in chunks(data) if kind == b"IDAT")


def filtered(m, types=None):
    """The filtered bytes of an 8-bit map with filter type 0 on every row (or ``types[y]``, the bytes left as they are)."""
    h, w = m.shape
    rows = np.zeros((h, w + 1), np.uint8)
    rows[:, 1:] = m
    if types is not None:
        rows[:, 0] = types
    return rows.tobytes()


def pillow(m, mode="L", **kw):
    from PIL import Image
    buf = io.BytesIO()
    img = Image.fromarray(m, "L")
    (img.convert("1") if mode == "1" else img).save(buf, "PNG", **kw)
    return buf.getvalue()


def opencv(m, level=None, strategy=None, bilevel=False):
    import cv2
    params = []
    if level is not None:
        params += [cv2.IMWRITE_PNG_COMPRESSION, level]
    if strategy is not None:
        params += [cv2.IMWRITE_PNG_STRATEGY, strategy]
    if bilevel:
        params += [cv2.IMWRITE_PNG_BILEVEL, 1]
    ok, buf = cv2.imencode(".png", m, params)
    assert ok
    return buf.tobytes()


def writers():
    import cv2
    return [("pillow", lambda m: pillow(m)),
            ("pillow-1", lambda m: pillow(m, "1")),
            ("pillow-level1", lambda m: pillow(m, compress_level=1)),
            ("pillow-level9", lambda m: pillow(m, compress_level=9)),
            ("pillow-optimize", lambda m: pillow(m, optimize=True)),
            ("cv2", lambda m: opencv(m)),
            ("cv2-level0", lambda m: opencv(m, 0)),
            ("cv2-level1", lambda m: opencv(m, 1)),
            ("cv2-level9", lambda m: opencv(m, 9)),
            ("cv2-fixed", lambda m: opencv(m, 9, cv2.IMWRITE_PNG_STRATEGY_FIXED)),
            ("cv2-huffman-only", lambda m: opencv(m, 6, cv2.IMWRITE_PNG_STRATEGY_HUFFMAN_ONLY)),
            ("cv2-rle", lambda m: opencv(m, 6, cv2.IMWRITE_PNG_STRATEGY_RLE)),
            ("cv2-bilevel", lambda m: opencv(m, bilevel=True)),
            ("own", lambda m: P.encode(m))]


def subset_files(shapes=None):
    """[(name, file bytes)] inside the device subset: every shape with rotating writers and contents, and every writer
    on one mid-sized shape."""
    out = []
    ws = writers()
    for i, (h, w) in enumerate(SHAPES if shapes is None else shapes):
        for j in range(3):
            name, fn = ws[(3 * i + j) % len(ws)]
            kind = C.KINDS[(i + j) % len(C.KINDS)]
            out.append((f"{name}-{kind}-{h}x{w}", fn(C.content(kind, h, w, seed=i))))
    for name, fn in ws:
        for kind in ("bytescale", "noise"):
            out.append((f"{name}-{kind}-40x56", fn(C.content(kind, 40, 56, seed=7))))
    return out


def full_flush_file(h=40, w=56, pieces=4, seed=1):
    """zlib's own Z_FULL_FLUSH between groups of rows, one IDAT per piece: true cuts from a foreign encoder, with real
    LZ77 matches inside each piece."""
    m = C.bytescale(h, w, seed)
    raw = filtered(m)
    co = zlib.compressobj(6)
    step = -(-h // pieces) * (w + 1)
    idats = []
    for k in range(0, len(raw), step):
        last = k + step >= len(raw)
        idats.append(co.compress(raw[k:k + step]) + co.flush(zlib.Z_FINISH if last else zlib.Z_FULL_FLUSH))
    return build(h, w, idats), m


def sync_flush_file(h=24, w=50, seed=2):
    """Z_SYNC_FLUSH half way, the second half repeating the first: the first IDAT ends in 00 00 FF FF, but the matches
    of the second reach back across it."""
    half = C.noise(h // 2, w, seed)
    m = np.concatenate([half, half])
    raw = filtered(m)
    co = zlib.compressobj(6)
    a = co.compress(raw[:len(raw) // 2]) + co.flush(zlib.Z_SYNC_FLUSH)
    b = co.compress(raw[len(raw) // 2:]) + co.flush()
    assert a.endswith(FLUSH)
    return build(h, w, [a, b]), m


def false_cut_file(h=12, w=40, seed=3):
    """One stored block whose pixel bytes contain 00 00 FF FF, the IDAT split right after them: a proposed cut inside
    a block."""
    m = C.noise(h, w, seed)
    m[5, 10:14] = [0, 0, 255, 255]
    stream = zlib.compress(filtered(m), 0)
    at = stream.index(FLUSH, 8) + 4
    return build(h, w, [stream[:at], stream[at:]]), m


def fallback_files():
    """{reason: file bytes} outside the subset, and the ones cv2 still reads."""
    from PIL import Image

    def save(img, **kw):
        buf = io.BytesIO()
        img.save(buf, "PNG", **kw)
        return buf.getvalue()
    m = C.bytescale(9, 11, 5)
    good = pillow(m)
    bad_crc = bytearray(good)
    bad_crc[-13] ^= 1                                          # the last IDAT's CRC
    one = zlib.compress(bytes([0, 77]))
    fdict = zlib.compressobj(6, zlib.DEFLATED, 15, 8, zlib.Z_DEFAULT_STRATEGY, b"\x00" * 12)
    return {
        "palette": save(Image.fromarray(m, "L").convert("P")),
        "RGB": save(Image.fromarray(np.stack([m] * 3, -1), "RGB")),
        "RGBA": save(Image.fromarray(np.stack([m] * 4, -1), "RGBA")),
        "gray+alpha": save(Image.fromarray(np.stack([m] * 2, -1), "LA")),
        "16-bit": save(Image.fromarray(m.astype(np.uint16) * 257)),
        "interlaced": build(1, 1, [one], interlace=1),
        "tRNS": build(9, 11, [zlib.compress(filtered(m))], extra=[(b"tRNS", b"\x00\x05")]),
        "bad CRC": bytes(bad_crc),
        "truncated": good[:len(good) - 20],
        "zlib preset dictionary": build(9, 11, [fdict.compress(filtered(m)) + fdict.flush()]),
        "not a PNG (no signature)": b"JFIF" + good[4:],
    }


CV2_READS = ["palette", "RGB", "RGBA", "gray+alpha", "16-bit", "interlaced", "tRNS"]


def corrupt_files(h=6, w=10, seed=4):
    """{status bit: (file bytes with valid chunk CRCs, so png.parse accepts it)}."""
    m = C.noise(h, w, seed)
    stored = zlib.compress(filtered(m), 0)
    flipped = bytearray(stored)
    flipped[2 + 5 + 3 * (w + 1) + 4] ^= 0x10                   # a pixel byte of row 3
    bad_filter = zlib.compress(filtered(m, types=[0, 0, 7, 0, 0, 0]), 6)
    # a final fixed-Huffman block whose first token is a match: BFINAL 1, BTYPE 01, length code 257 (0000001),
    # distance code 0 (00000): bits, LSB first, 1 10 0000001 00000
    bits = [1, 1, 0] + [0, 0, 0, 0, 0, 0, 1] + [0] * 5
    body = bytearray((len(bits) + 7) // 8)
    for i, v in enumerate(bits):
        body[i >> 3] |= v << (i & 7)
    return {
        4: build(h, w, [stored[:len(stored) // 2]]),
        8: build(h, w, [bytes(flipped)]),
        16: build(h, w, [bad_filter]),
        2: build(h, w, [b"\x78\x01" + bytes(body) + b"\x00\x00\x00\x01"]),
        1: build(h, w, [b"\x78\x01\x07\x00" + b"\x00\x00\x00\x01"]),
    }, m
