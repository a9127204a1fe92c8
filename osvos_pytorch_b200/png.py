"""Host side of the device PNG decoder (csrc/png_decode.cu, DESIGN.md §22): chunk parsing and batch packing, no pixel
work.

``parse(data)`` walks a PNG file's chunks and returns a ``Parsed`` description, or a ``Fallback`` naming why the file
is outside the subset the device decodes: colour type 0 (grayscale), bit depth 8 or 1, no interlace, no ``tRNS``; any
ancillary chunks, any split of the zlib stream over ``IDAT`` chunks.  Everything else is decoded by
``cv2.imdecode(..., 0)`` on the host.  Bit depth 1 decodes to 0 / 255, as cv2 gives.

``parse(data, palette="index")`` (DAVIS-2017 label files, DESIGN.md §24) also accepts colour type 3 (palette) at bit
depths 1, 2, 4 and 8, with or without ``tRNS`` (transparency does not change the indices); the device writes each
pixel's raw index, what ``np.array(PIL.Image.open(f))`` gives.  In that mode the host fallback is Pillow, never cv2,
whose conversion to gray would lose the indices.

Proposed cuts: a zlib stream can be inflated in independent pieces where a full flush happened: the stream is on a
byte boundary there, the bytes before it are ``00 00 FF FF`` and no match reaches back across it.  The project's own
encoder (csrc/png.cu) ends every ``IDAT`` that way.  ``parse`` proposes a cut after every ``IDAT`` payload that ends
in those four bytes.  That is a hint, not a proof (another encoder may end a chunk on them by chance, and a sync flush
leaves matches that cross); the kernels prove or reject the cuts of each file and a rejected file is inflated in
order, so a wrong hint changes neither pixels nor status.

``pack(parsed_list)`` lays a batch of one size out as one uint8 blob (one host-to-device copy):

    HEADER   magic "PNG1", n, nseg, h, w, 3 pad | offsets of the file table, the segment table and the data, data bytes
    FILE     per file: h, w, depth, first segment, segment count, 3 pad | offset and length of its zlib stream in the data
    SEGMENT  per segment: [beg, end) in the data | file, index in the file.  Segment 0 begins after the 2-byte zlib
             header, the last one ends with the 4 Adler-32 bytes
    data     the zlib streams (the concatenated IDAT payloads), back to back

every table 16-byte aligned.  The structs at the top of csrc/png_decode.cu mirror it.
"""
import struct
import zlib
from dataclasses import dataclass, field

import numpy as np

MAGIC = 0x31474E50                      # "PNG1"
HEADER = struct.Struct("<8i4q")
FILE = np.dtype([("h", "<i4"), ("w", "<i4"), ("depth", "<i4"), ("seg0", "<i4"), ("nseg", "<i4"), ("colour", "<i4"),
                 ("pad", "<i4", 2),
                 ("stream_off", "<i8"), ("stream_len", "<i8")])
SEGMENT = np.dtype([("beg", "<i8"), ("end", "<i8"), ("file", "<i4"), ("index", "<i4")])
SIGNATURE = b"\x89PNG\r\n\x1a\n"
FLUSH = b"\x00\x00\xff\xff"
_COLOUR = {2: "RGB", 3: "palette", 4: "gray+alpha", 6: "RGBA"}


@dataclass
class Fallback:
    """A file outside the device subset; ``reason`` says why."""
    reason: str


@dataclass
class Parsed:
    """A PNG inside the device subset."""
    h: int
    w: int
    depth: int
    stream: bytes                                   # the zlib stream: the IDAT payloads concatenated
    cuts: list = field(default_factory=list)        # proposed segment starts after the first, offsets in ``stream``
    colour: int = 0                                 # PNG colour type: 0 grayscale, 3 palette
    palette: bytes = None                           # the PLTE chunk's bytes (RGB triples) of a palette file

    @property
    def rowbytes(self):
        return -(-self.w * self.depth // 8)


def parse(data, palette=None):
    """Parse a PNG file's bytes -> Parsed, or Fallback(reason) for a file outside the device subset.  ``palette``:
    None (grayscale files only) or "index" (palette files too, decoded to their indices)."""
    if palette not in (None, "index"):
        raise ValueError(f"palette must be None or 'index', got {palette!r}")
    data = bytes(data)
    if data[:8] != SIGNATURE:
        return Fallback("not a PNG (no signature)")
    p, n = 8, len(data)
    ihdr = None
    payloads = []
    plte = trns = None
    ended = False
    while p < n:
        if p + 12 > n:
            return Fallback("truncated")
        ln, = struct.unpack(">I", data[p:p + 4])
        kind = data[p + 4:p + 8]
        if p + 12 + ln > n:
            return Fallback("truncated")
        body = data[p + 8:p + 8 + ln]
        if zlib.crc32(data[p + 4:p + 8 + ln]) != struct.unpack(">I", data[p + 8 + ln:p + 12 + ln])[0]:
            return Fallback("bad CRC")
        p += 12 + ln
        if ihdr is None:
            if kind != b"IHDR" or ln != 13:
                return Fallback("no IHDR")
            ihdr = struct.unpack(">IIBBBBB", body)
        elif kind == b"IDAT":
            payloads.append(body)
        elif kind == b"PLTE":
            plte = body
        elif kind == b"tRNS":
            trns = body
        elif kind == b"IEND":
            ended = True
            break
    if ihdr is None or not ended:
        return Fallback("truncated")
    w, h, depth, colour, compression, filtering, interlace = ihdr
    if colour == 3 and palette == "index":
        if depth not in (1, 2, 4, 8):
            return Fallback(f"{depth}-bit")
        if plte is None or not plte or len(plte) % 3 or len(plte) > 768:
            return Fallback("no valid PLTE")
    else:
        if colour != 0:
            return Fallback(_COLOUR.get(colour, f"colour type {colour}"))
        if trns is not None:
            return Fallback("tRNS")
        if depth not in (1, 8):
            return Fallback(f"{depth}-bit")
    if interlace != 0:
        return Fallback("interlaced")
    if compression != 0 or filtering != 0:
        return Fallback("compression or filter method")
    if not (0 < h < 32768 and 0 < w < 32768):
        return Fallback("size")
    stream = b"".join(payloads)
    if len(stream) < 6:
        return Fallback("truncated")
    cmf, flg = stream[0], stream[1]
    if (cmf & 15) != 8 or (cmf >> 4) > 7 or ((cmf << 8) | flg) % 31:
        return Fallback("zlib header")
    if flg & 32:
        return Fallback("zlib preset dictionary")
    cuts, at = [], 0
    for body in payloads[:-1]:
        at += len(body)
        if at >= 6 and at < len(stream) and stream[at - 4:at] == FLUSH and (not cuts or cuts[-1] != at):
            cuts.append(at)
    return Parsed(h, w, depth, stream, cuts, colour, plte if colour == 3 else None)


def pack(parsed_list):
    """One uint8 numpy blob holding a batch of Parsed files of one size (layout: module docstring)."""
    if not parsed_list:
        raise ValueError("pack needs at least one file")
    h, w = parsed_list[0].h, parsed_list[0].w
    if any((p.h, p.w) != (h, w) for p in parsed_list):
        raise ValueError("all files of a blob share one size, got " + ", ".join(sorted({f"{p.h}x{p.w}" for p in parsed_list})))
    files = np.zeros(len(parsed_list), FILE)
    segs = []
    off = 0
    for i, p in enumerate(parsed_list):
        bounds = [2] + list(p.cuts) + [len(p.stream)]
        files[i] = (h, w, p.depth, len(segs), len(bounds) - 1, p.colour, 0, off, len(p.stream))
        segs.extend((off + bounds[k], off + bounds[k + 1], i, k) for k in range(len(bounds) - 1))
        off += len(p.stream)
    parts = [files.tobytes(), np.array(segs, dtype=SEGMENT).tobytes()]
    offs, o = [], HEADER.size
    for part in parts:
        offs.append(o)
        o += -(-len(part) // 16) * 16
    blob = np.zeros(o + off, np.uint8)
    blob[:HEADER.size] = np.frombuffer(HEADER.pack(MAGIC, len(parsed_list), len(segs), h, w, 0, 0, 0, *offs, o, off),
                                       np.uint8)
    for at, part in zip(offs, parts):
        blob[at:at + len(part)] = np.frombuffer(part, np.uint8)
    blob[o:] = np.frombuffer(b"".join(p.stream for p in parsed_list), np.uint8)
    return blob


def segment_count(blob):
    """The number of segments in a packed blob (its header's nseg)."""
    return int(HEADER.unpack_from(bytes(blob[:HEADER.size]))[2])


def decode_host(data):
    """One file's bytes -> uint8 [h, w] as cv2.imread(path, 0) gives."""
    import cv2
    m = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_GRAYSCALE)
    if m is None:
        raise ValueError("cv2 cannot decode this PNG")
    return m


def decode_host_index(data):
    """One file's bytes -> uint8 [h, w] as np.array(PIL.Image.open(f)) gives: a palette file's indices, a grayscale
    file's values (depth 1 as 0 / 255).  Other colour types raise ValueError."""
    import io

    from PIL import Image
    img = Image.open(io.BytesIO(bytes(data)))
    if img.mode == "1":
        img = img.convert("L")
    if img.mode not in ("P", "L"):
        raise ValueError(f"an index or grayscale PNG is needed, got mode {img.mode}")
    return np.array(img, dtype=np.uint8)


def palette_of(data):
    """The PLTE chunk's bytes (RGB triples) of a PNG file, or None when it has none."""
    data = bytes(data)
    p = 8
    while p + 8 <= len(data):
        ln, = struct.unpack(">I", data[p:p + 4])
        kind = data[p + 4:p + 8]
        if kind == b"PLTE":
            return data[p + 8:p + 8 + ln]
        if kind in (b"IDAT", b"IEND"):
            return None
        p += 12 + ln
    return None


def decode_files(datas, device, parsed=None, palette=None):
    """A list of PNG files' bytes, all of one size -> (uint8 [n,h,w] on ``device``, fallback count, re-decoded count).

    Files inside the subset are decoded on the device (ops.decode_png); Fallback files, and after one read of the
    status words the files the decoder flagged, are decoded by cv2 on the host (Pillow with ``palette="index"``,
    see ``parse``).  ``parsed``: the files' ``parse`` results when the caller has them already (reader threads)."""
    import torch

    from . import ops
    if parsed is None:
        parsed = [parse(d, palette=palette) for d in datas]
    host_decode = decode_host_index if palette == "index" else decode_host
    n = len(datas)
    sub = [i for i, p in enumerate(parsed) if isinstance(p, Parsed)]
    host = {i: host_decode(datas[i]) for i in range(n) if not isinstance(parsed[i], Parsed)}
    fallback = len(host)
    sizes = {(parsed[i].h, parsed[i].w) for i in sub} | {m.shape for m in host.values()}
    if len(sizes) != 1:
        raise ValueError("the files differ in size: " + ", ".join(f"{a}x{b}" for a, b in sorted(sizes)))
    (h, w), = sizes
    out = torch.empty((n, h, w), dtype=torch.uint8, device=device)
    if sub:
        blob = pack([parsed[i] for i in sub])
        dev_blob = torch.from_numpy(blob).to(device)
        got, status = ops.decode_png(dev_blob, len(sub), h, w, segment_count(blob), out=out if len(sub) == n else None)
        if len(sub) != n:
            out[torch.tensor(sub, device=device)] = got
        for j in torch.nonzero(status.cpu()).flatten().tolist():
            host[sub[j]] = host_decode(datas[sub[j]])
            if host[sub[j]].shape != (h, w):
                raise ValueError("the files differ in size")
    if host:
        idx = sorted(host)
        out[torch.tensor(idx, device=device)] = torch.from_numpy(np.stack([host[i] for i in idx])).to(device)
    return out, fallback, len(host) - fallback
