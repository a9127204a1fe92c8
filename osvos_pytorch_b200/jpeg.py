"""Host side of the device JPEG decoder (csrc/jpeg.cu, DESIGN.md §19): marker parsing and batch packing, no pixel work.

``parse(buf)`` walks a JPEG file's markers and returns a ``Parsed`` description of the image, or a ``Fallback`` naming
why the file is outside the subset the device decodes bit-identically to ``cv2.imread`` (libjpeg-turbo: ISLOW integer
IDCT, fancy upsampling, fixed-point YCbCr -> BGR).  The subset: SOF0 / SOF1, 8-bit, Huffman, one scan; one component,
or three in one interleaved scan with luma sampling (1,1), (2,1), (1,2) or (2,2) and chroma (1,1); any restart
interval; YCbCr as libjpeg decides it (JFIF marker, Adobe transform, component IDs); no EXIF rotation.  Everything else
is decoded by ``cv2.imread`` as before.

``pack(parsed_list)`` lays a batch out as one uint8 blob (one host-to-device copy): a header, per-image headers,
segment descriptors, quantisation tables in natural order, Huffman lookup tables and the de-stuffed entropy-coded
segments (split at RST markers).  The layout is mirrored by the structs at the top of csrc/jpeg.cu.
"""
import struct
from dataclasses import dataclass, field

import numpy as np

MAGIC = 0x3147504A                      # "JPG1"
HEADER = struct.Struct("<8i6q")         # magic, n, nseg, nq, nh, 3 x pad | img, seg, q, huff, data offsets, data bytes
IMAGE_INTS = 24                         # h, w, ncomp, hs, vs, mcux, mcuy, bpm, restart, seg0, nseg, q[3], dc[3], ac[3]
SEGMENT = np.dtype([("byte_off", "<i8"), ("nbits", "<i8"), ("image", "<i4"), ("first_block", "<i4"),
                    ("nblocks", "<i4"), ("pad", "<i4")])
LOOKAHEAD = 9
HUFF = np.dtype([("lookup", "<u2", 1 << LOOKAHEAD), ("maxcode", "<i4", 18), ("valoffset", "<i4", 18),
                 ("vals", "u1", 256)])

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                   6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45,
                   38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63], dtype=np.int32)   # zig-zag index -> natural index


@dataclass
class Fallback:
    """A file outside the device subset; ``reason`` says why."""
    reason: str


@dataclass
class Huffman:
    lookup: np.ndarray                 # [512] (length << 8) | symbol for codes of <= 9 bits, else (10 << 8)
    maxcode: np.ndarray                # [18] libjpeg's maxcode (maxcode[17] = 0xFFFFF)
    valoffset: np.ndarray              # [18]
    vals: np.ndarray                   # [256]


@dataclass
class Parsed:
    """A JPEG inside the device subset."""
    h: int
    w: int
    ncomp: int
    hs: int                             # luma sampling (chroma is (1, 1)); (1, 1) for one component
    vs: int
    restart: int                        # MCUs per restart interval (0: none)
    qt: list                            # per component: uint16 [64] in natural order
    dc: list                            # per component: Huffman
    ac: list
    segments: list = field(default_factory=list)   # de-stuffed entropy-coded bytes, one per restart interval

    @property
    def bpm(self):
        return self.hs * self.vs + 2 if self.ncomp == 3 else 1

    @property
    def mcux(self):
        return -(-self.w // (8 * self.hs))

    @property
    def mcuy(self):
        return -(-self.h // (8 * self.vs))


def huffman_table(bits, vals):
    """libjpeg's jpeg_make_d_derived_tbl for BITS[1..16] and HUFFVAL; None for a table libjpeg rejects."""
    sizes = [l for l in range(1, 17) for _ in range(bits[l - 1])]
    if len(sizes) > 256 or len(sizes) != len(vals):
        return None
    codes, code, si, p = [], 0, sizes[0] if sizes else 0, 0
    while p < len(sizes):
        while p < len(sizes) and sizes[p] == si:
            codes.append(code)
            code += 1
            p += 1
        if code >= (1 << si):
            return None
        code <<= 1
        si += 1
    maxcode = np.full(18, -1, np.int32)
    valoffset = np.zeros(18, np.int32)
    p = 0
    for l in range(1, 17):
        if bits[l - 1]:
            valoffset[l] = p - codes[p]
            p += bits[l - 1]
            maxcode[l] = codes[p - 1]
    maxcode[17] = 0xFFFFF
    lookup = np.full(1 << LOOKAHEAD, (LOOKAHEAD + 1) << 8, np.uint16)
    p = 0
    for l in range(1, LOOKAHEAD + 1):
        for _ in range(bits[l - 1]):
            base = codes[p] << (LOOKAHEAD - l)
            lookup[base:base + (1 << (LOOKAHEAD - l))] = (l << 8) | vals[p]
            p += 1
    v = np.zeros(256, np.uint8)
    v[:len(vals)] = vals
    return Huffman(lookup, maxcode, valoffset, v)


def _exif_orientation(d):
    """The TIFF orientation tag of an APP1 'Exif' payload (bytes after 'Exif\\0\\0'), or 1."""
    if len(d) < 8 or d[:2] not in (b"II", b"MM"):
        return 1
    e = "<" if d[:2] == b"II" else ">"
    ifd = struct.unpack(e + "I", d[4:8])[0]
    if ifd + 2 > len(d):
        return 1
    for i in range(struct.unpack(e + "H", d[ifd:ifd + 2])[0]):
        o = ifd + 2 + 12 * i
        if o + 12 > len(d):
            break
        if struct.unpack(e + "H", d[o:o + 2])[0] == 0x0112:
            return struct.unpack(e + "H", d[o + 8:o + 10])[0]
    return 1


_SOF_NAMES = {0xC2: "progressive", 0xC3: "lossless", 0xC5: "hierarchical", 0xC6: "hierarchical", 0xC7: "hierarchical",
              0xC9: "arithmetic", 0xCA: "arithmetic", 0xCB: "arithmetic", 0xCD: "arithmetic", 0xCE: "arithmetic",
              0xCF: "arithmetic"}


def _split_scan(a, p):
    """De-stuff the entropy-coded data from a[p:] as libjpeg's bit reader reads it, split at RST markers.  Returns
    (segments, RST numbers seen in order, position of the marker that ends the scan or len(a)).

    A run of FF bytes is fill before the byte after it: 00 makes the run one FF data byte, D0-D7 is a restart
    boundary, anything else (or the end of the buffer) ends the scan.  All of it with numpy: no per-byte Python."""
    b = a[p:]
    n = len(b)
    ff = np.flatnonzero(b == 0xFF)
    if len(ff) == 0:
        return [b.tobytes()], [], len(a)
    first = np.concatenate([[True], np.diff(ff) != 1])
    starts = ff[first]                                   # first FF of each run
    j = np.concatenate([ff[np.flatnonzero(first)[1:] - 1], ff[-1:]]) + 1               # the byte after each run
    follow = np.where(j < n, b[np.minimum(j, n - 1)], -1).astype(np.int32)
    stuffed = follow == 0
    rst = (follow >= 0xD0) & (follow <= 0xD7)
    term = ~(stuffed | rst)
    end = n
    if term.any():
        t = int(np.argmax(term))
        end = int(starts[t])
        starts, j, follow, stuffed, rst = starts[:t], j[:t], follow[:t], stuffed[:t], rst[:t]
    lo = np.where(stuffed, starts + 1, starts)           # dropped: [lo, j] (the fill FFs and the 00, or the marker)
    lens = j + 1 - lo
    drop = np.repeat(lo - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens) + np.arange(int(lens.sum()))
    keep = np.ones(end, bool)
    keep[drop[drop < end]] = False
    cut = starts[rst]
    segments = np.split(b[:end][keep], cut - np.searchsorted(drop, cut))
    return [seg.tobytes() for seg in segments], [int(v) - 0xD0 for v in follow[rst]], p + end


def parse(buf):
    """Parse a JPEG file's bytes -> Parsed, or Fallback(reason) for a file outside the device subset."""
    a = np.frombuffer(bytes(buf), dtype=np.uint8)
    n = len(a)
    if n < 4 or a[0] != 0xFF or a[1] != 0xD8:
        return Fallback("not a JPEG (no SOI)")
    qt, dc, ac = {}, {}, {}
    frame = None
    restart = 0
    jfif = adobe = False
    adobe_transform = -1
    p = 2
    while True:
        while p < n and a[p] != 0xFF:                # libjpeg skips garbage before a marker
            p += 1
        while p < n and a[p] == 0xFF:
            p += 1
        if p >= n:
            return Fallback("truncated headers")
        m = int(a[p])
        p += 1
        if m == 0xD8 or 0xD0 <= m <= 0xD7 or m == 0x01:
            continue
        if m == 0xD9:
            return Fallback("no SOS")
        if p + 2 > n:
            return Fallback("truncated headers")
        ln = (int(a[p]) << 8) | int(a[p + 1])
        if ln < 2 or p + ln > n:
            return Fallback("truncated headers")
        d = a[p + 2:p + ln].tobytes()
        p += ln
        if m == 0xE0 and d[:5] == b"JFIF\0":
            jfif = True
        elif m == 0xEE and d[:5] == b"Adobe" and len(d) >= 12:
            adobe, adobe_transform = True, d[11]
        elif m == 0xE1 and d[:6] == b"Exif\0\0":
            if _exif_orientation(d[6:]) != 1:
                return Fallback("EXIF orientation")
        elif m == 0xDB:
            q = 0
            while q < len(d):
                pq, tq = d[q] >> 4, d[q] & 15
                size = 128 if pq else 64
                if tq > 3 or q + 1 + size > len(d):
                    return Fallback("bad DQT")
                vals = np.frombuffer(d[q + 1:q + 1 + size], dtype=">u2" if pq else np.uint8).astype(np.uint16)
                t = np.zeros(64, np.uint16)
                t[ZIGZAG] = vals
                qt[tq] = t
                q += 1 + size
        elif m == 0xC4:
            q = 0
            while q < len(d):
                if q + 17 > len(d):
                    return Fallback("bad DHT")
                tc, th = d[q] >> 4, d[q] & 15
                bits = list(d[q + 1:q + 17])
                cnt = sum(bits)
                vals = list(d[q + 17:q + 17 + cnt])
                if tc > 1 or th > 3 or len(vals) != cnt or (tc == 0 and any(v > 15 for v in vals)):
                    return Fallback("bad DHT")
                tab = huffman_table(bits, vals)
                if tab is None:
                    return Fallback("bad DHT")
                (ac if tc else dc)[th] = tab
                q += 17 + cnt
        elif m == 0xDD:
            if len(d) < 2:
                return Fallback("bad DRI")
            restart = (d[0] << 8) | d[1]
        elif m == 0xCC:
            return Fallback("arithmetic")
        elif m in _SOF_NAMES:
            return Fallback(_SOF_NAMES[m])
        elif m in (0xC0, 0xC1):
            if frame is not None:
                return Fallback("two frames")
            if len(d) < 6 or d[0] != 8:
                return Fallback("precision") if len(d) >= 1 and d[0] != 8 else Fallback("truncated headers")
            h, w, nf = (d[1] << 8) | d[2], (d[3] << 8) | d[4], d[5]
            if len(d) < 6 + 3 * nf:
                return Fallback("truncated headers")
            comps = [(d[6 + 3 * i], d[7 + 3 * i] >> 4, d[7 + 3 * i] & 15, d[8 + 3 * i]) for i in range(nf)]
            frame = (h, w, comps)
        elif m == 0xDA:
            break
    if frame is None:
        return Fallback("no frame header")
    h, w, comps = frame
    if h == 0 or w == 0:
        return Fallback("DNL")
    if len(comps) not in (1, 3):
        return Fallback(f"{len(comps)} components")
    if len(comps) == 3:
        ids = [c[0] for c in comps]
        if jfif:
            pass
        elif adobe:
            if adobe_transform == 0:
                return Fallback("RGB (Adobe transform 0)")
        elif ids == [82, 71, 66]:
            return Fallback("RGB component IDs")
        samp = [(c[1], c[2]) for c in comps]
        if samp[1] != (1, 1) or samp[2] != (1, 1) or samp[0] not in ((1, 1), (2, 1), (1, 2), (2, 2)):
            return Fallback("sampling " + ",".join(f"{a}x{b}" for a, b in samp))
        hs, vs = samp[0]
    else:
        hs = vs = 1                                  # a one-component scan is not interleaved: one block per MCU
    if len(d) < 1 or len(d) < 1 + 2 * d[0] + 3:
        return Fallback("truncated headers")
    ns = d[0]
    if ns != len(comps):
        return Fallback("multi-scan")
    sel = [(d[1 + 2 * i], d[2 + 2 * i] >> 4, d[2 + 2 * i] & 15) for i in range(ns)]
    ss, se, ahal = d[1 + 2 * ns], d[2 + 2 * ns], d[3 + 2 * ns]
    if (ss, se, ahal) != (0, 63, 0):
        return Fallback("spectral selection")
    if [s[0] for s in sel] != [c[0] for c in comps]:
        return Fallback("scan component order")
    try:
        q = [qt[c[3]] for c in comps]
        dct = [dc[s[1]] for s in sel]
        act = [ac[s[2]] for s in sel]
    except KeyError:
        return Fallback("missing table")
    segments, rsts, end = _split_scan(a, p)
    mcus = -(-w // (8 * hs)) * -(-h // (8 * vs))
    want = 1 if restart == 0 else -(-mcus // restart)
    if len(segments) != want or any(r != i % 8 for i, r in enumerate(rsts)):
        return Fallback("restart markers")
    # one scan only: a second SOS after this one is a multi-scan file
    p = end
    while p + 1 < n:
        while p < n and a[p] != 0xFF:
            p += 1
        while p < n and a[p] == 0xFF:
            p += 1
        if p >= n:
            break
        m2 = int(a[p])
        if m2 == 0xD9:
            break
        if m2 in (0xDA, 0xDC):
            return Fallback("multi-scan" if m2 == 0xDA else "DNL")
        if 0xD0 <= m2 <= 0xD7 or m2 == 0x01 or p + 3 > n:
            p += 1
            continue
        p += 1 + ((int(a[p + 1]) << 8) | int(a[p + 2]))
    return Parsed(h, w, len(comps), hs, vs, restart, q, dct, act, segments)


def pack(parsed_list):
    """One uint8 numpy blob holding a batch of Parsed images (layout: module docstring and csrc/jpeg.cu)."""
    qs, hts, qid, hid = [], [], {}, {}

    def table(store, index, key, value):
        if key not in index:
            index[key] = len(store)
            store.append(value)
        return index[key]

    imgs = np.zeros((len(parsed_list), IMAGE_INTS), np.int32)
    segs, datas = [], []
    data_off = 0
    for i, pj in enumerate(parsed_list):
        q = [table(qs, qid, t.tobytes(), t) for t in pj.qt]
        dc = [table(hts, hid, ("d", t.lookup.tobytes(), t.vals.tobytes()), t) for t in pj.dc]
        ac = [table(hts, hid, ("a", t.lookup.tobytes(), t.vals.tobytes(), t.maxcode.tobytes()), t) for t in pj.ac]
        pad = [0] * (3 - pj.ncomp)
        bpm = pj.bpm
        per_seg = pj.restart if pj.restart else pj.mcux * pj.mcuy
        imgs[i] = [pj.h, pj.w, pj.ncomp, pj.hs, pj.vs, pj.mcux, pj.mcuy, bpm, per_seg, len(segs), len(pj.segments)] \
            + q + pad + dc + pad + ac + pad + [0] * 4
        total = pj.mcux * pj.mcuy * bpm
        for s, seg in enumerate(pj.segments):
            first = s * per_seg * bpm
            segs.append((data_off, 8 * len(seg), i, first, min(per_seg * bpm, total - first), 0))
            datas.append(seg)
            data_off += len(seg)
    seg_arr = np.array(segs, dtype=SEGMENT)
    q_arr = np.array(qs, dtype=np.uint16).reshape(-1, 64)
    h_arr = np.zeros(len(hts), dtype=HUFF)
    for k, t in enumerate(hts):
        h_arr[k] = (t.lookup, t.maxcode, t.valoffset, t.vals)
    parts = [imgs.tobytes(), seg_arr.tobytes(), q_arr.tobytes(), h_arr.tobytes()]
    offs, o = [], HEADER.size
    for part in parts:
        offs.append(o)
        o += -(-len(part) // 16) * 16
    data = b"".join(datas)
    blob = np.zeros(o + len(data), np.uint8)
    blob[:HEADER.size] = np.frombuffer(HEADER.pack(MAGIC, len(parsed_list), len(segs), len(qs), len(hts), 0, 0, 0,
                                                   *offs, o, len(data)), np.uint8)
    for off, part in zip(offs, parts):
        blob[off:off + len(part)] = np.frombuffer(part, np.uint8)
    blob[o:] = np.frombuffer(data, np.uint8)
    return blob


def segment_count(blob):
    """The number of entropy-coded segments in a packed blob (its header's nseg)."""
    return int(HEADER.unpack_from(bytes(blob[:HEADER.size]))[2])


def decode_host(data):
    """One file's bytes -> uint8 [h, w, 3] BGR as cv2.imread(path) gives."""
    import cv2
    img = cv2.imdecode(np.frombuffer(bytes(data), np.uint8), cv2.IMREAD_COLOR)
    if img is None:
        raise ValueError("cv2 cannot decode this JPEG")
    return img


def decode_files(datas, device, parsed=None):
    """A list of JPEG files' bytes, all of one size -> (uint8 [n,h,w,3] BGR on ``device``, fallback count, re-decoded
    count), bit-identical to cv2.imread.

    Files inside the subset are decoded on the device (ops.decode_jpeg); Fallback files, and after one read of the
    status words the files the decoder flagged, are decoded by cv2 on the host.  ``parsed``: the files' ``parse``
    results when the caller has them already (reader threads).  png.decode_files is the same for PNGs."""
    import torch

    from . import ops
    if parsed is None:
        parsed = [parse(d) for d in datas]
    n = len(datas)
    sub = [i for i, p in enumerate(parsed) if isinstance(p, Parsed)]
    host = {i: decode_host(datas[i]) for i in range(n) if not isinstance(parsed[i], Parsed)}
    fallback = len(host)
    sizes = {(parsed[i].h, parsed[i].w) for i in sub} | {m.shape[:2] for m in host.values()}
    if len(sizes) != 1:
        raise ValueError("the files differ in size: " + ", ".join(f"{a}x{b}" for a, b in sorted(sizes)))
    (h, w), = sizes
    out = torch.empty((n, h, w, 3), dtype=torch.uint8, device=device)
    if sub:
        blob = pack([parsed[i] for i in sub])
        dev_blob = torch.from_numpy(blob).to(device)
        got, status = ops.decode_jpeg(dev_blob, len(sub), h, w, out=out if len(sub) == n else None,
                                      nseg=segment_count(blob))
        if len(sub) != n:
            out[torch.tensor(sub, device=device)] = got
        for j in torch.nonzero(status.cpu()).flatten().tolist():
            host[sub[j]] = decode_host(datas[sub[j]])
            if host[sub[j]].shape[:2] != (h, w):
                raise ValueError("the files differ in size")
    if host:
        idx = sorted(host)
        out[torch.tensor(idx, device=device)] = torch.from_numpy(np.stack([host[i] for i in idx])).to(device)
    return out, fallback, len(host) - fallback
