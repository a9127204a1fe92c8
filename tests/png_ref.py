"""numpy restatement of the device PNG encoder (csrc/png.cu, DESIGN.md §21), byte for byte, and a plain decoder.

encode(a) turns one uint8 map [H,W] into the exact file the kernels write; decode(data) inflates with zlib and undoes
the row filters in numpy, independently of Pillow and libpng.  Every format decision below is the one the kernels make:
  - rows are filtered with the type 0-4 of least sum(min(v, 256 - v)) over the filtered bytes, ties to the lower type;
  - the filtered stream is cut into segments of R = max(1, SEGMENT_BYTES // (W + 1)) rows; each segment is one IDAT
    chunk holding one dynamic-Huffman block or one stored block (whichever is smaller, stored on a tie), BFINAL 0,
    followed by an empty stored block (zlib's full flush); the first segment starts with the zlib header 78 01;
  - tokens are literals and distance-1 matches: a run of n >= 4 equal bytes is one literal, then matches of 258, then
    a remainder of 3..257 as one more match or 1..2 as literals;
  - Huffman lengths: two-queue Huffman over the used symbols sorted by (count, symbol), the per-length counts limited
    to 15 (7 for the code-length code) by moving codes down from the longest length (miniz's rule), lengths handed out
    in that order from the longest; canonical codes (RFC 1951); one distance code (symbol 0, one bit);
  - a trailer IDAT with a final empty fixed-Huffman block (03 00) and the Adler-32, then IEND."""
import struct
import zlib

import numpy as np

SEGMENT_BYTES = 16384
SIGNATURE = b"\x89PNG\r\n\x1a\n"
CL_ORDER = (16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15)


def max_bytes(h, w):
    """osvos_png_max_bytes: every segment stored."""
    if not (0 < h < 32768 and 0 < w < 32768):
        return 0
    rows = max(1, SEGMENT_BYTES // (w + 1))
    nseg = -(-h // rows)
    return 8 + 25 + 2 + 18 + 12 + 22 * nseg + h * (w + 1)


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_rows(a):
    """uint8 [H,W] -> (types [H], filtered stream [H, W+1] uint8 with the type byte first)."""
    a = np.asarray(a, dtype=np.int32)
    h, w = a.shape
    prior = np.vstack([np.zeros((1, w), np.int32), a[:-1]])
    left = np.hstack([np.zeros((h, 1), np.int32), a[:, :-1]])
    upleft = np.hstack([np.zeros((h, 1), np.int32), prior[:, :-1]])
    cand = np.stack([a, a - left, a - prior, a - (left + prior) // 2, a - _paeth(left, prior, upleft)]) & 255
    cost = np.minimum(cand, 256 - cand).sum(axis=2)                         # [5, H]
    types = np.argmin(cost, axis=0)                                         # first minimum: ties to the lower type
    out = np.empty((h, w + 1), np.uint8)
    out[:, 0] = types
    out[:, 1:] = cand[types, np.arange(h)]
    return types, out


def huffman_lengths(freq, maxlen):
    """Code lengths (list) for counts `freq`, limited to maxlen; see the module docstring."""
    syms = sorted((i for i in range(len(freq)) if freq[i] > 0), key=lambda i: (freq[i], i))
    nu = len(syms)
    assert nu >= 2, "every code here has at least two symbols"
    lw = [freq[s] for s in syms]
    iw, ipar, lpar = [], [], [0] * nu
    li = ii = 0
    for k in range(nu - 1):
        w = 0
        for _ in range(2):
            if li < nu and (ii >= k or lw[li] <= iw[ii]):
                w += lw[li]
                lpar[li] = k
                li += 1
            else:
                w += iw[ii]
                ipar[ii] = k
                ii += 1
        iw.append(w)
        ipar.append(-1)
    idepth = [0] * (nu - 1)
    for k in range(nu - 3, -1, -1):
        idepth[k] = idepth[ipar[k]] + 1
    count = [0] * (maxlen + 1)
    for k in range(nu):
        count[min(idepth[lpar[k]] + 1, maxlen)] += 1
    total = sum(count[i] << (maxlen - i) for i in range(1, maxlen + 1))
    while total != 1 << maxlen:
        count[maxlen] -= 1
        for i in range(maxlen - 1, 0, -1):
            if count[i]:
                count[i] -= 1
                count[i + 1] += 2
                break
        total -= 1
    lengths = [0] * len(freq)
    pos = 0
    for ln in range(maxlen, 0, -1):
        for _ in range(count[ln]):
            lengths[syms[pos]] = ln
            pos += 1
    return lengths


def canonical_codes(lengths):
    """RFC 1951 canonical codes, bit-reversed for LSB-first packing."""
    maxlen = max(lengths)
    count = [0] * (maxlen + 1)
    for ln in lengths:
        if ln:
            count[ln] += 1
    nxt, code = [0] * (maxlen + 1), 0
    for b in range(1, maxlen + 1):
        code = (code + count[b - 1]) << 1 if b > 1 else 0
        nxt[b] = code
    out = [0] * len(lengths)
    for s, ln in enumerate(lengths):
        if ln:
            c = nxt[ln]
            nxt[ln] += 1
            out[s] = int(format(c, f"0{ln}b")[::-1], 2)
    return out


def length_symbol(r):
    """Match length r (3..258) -> (symbol, extra bit count, extra value)."""
    if r <= 10:
        return 254 + r, 0, 0
    if r == 258:
        return 285, 0, 0
    x = r - 3
    e = x.bit_length() - 3
    return 257 + 4 * (e + 1) + (x >> e) - 4, e, x & ((1 << e) - 1)


_LSYM = np.zeros(259, np.int64)
_LEXB = np.zeros(259, np.int64)
_LEXV = np.zeros(259, np.int64)
for _r in range(3, 259):
    _LSYM[_r], _LEXB[_r], _LEXV[_r] = length_symbol(_r)


def tokens(d):
    """Segment bytes -> (symbol, extra bits, extra value, match flag) arrays in stream order."""
    d = np.asarray(d, np.int64)
    starts = np.flatnonzero(np.r_[True, d[1:] != d[:-1]])
    n = np.diff(np.r_[starts, len(d)])
    v = d[starts]
    long_ = n >= 4
    m = n - 1
    q = np.where(long_, m // 258, 0)
    r = m % 258
    c = (long_ & (r >= 3)).astype(np.int64)
    a = np.where(long_, 1, n)
    b = np.where(long_ & (r < 3), r, 0)
    counts = np.stack([a, q, c, b], 1).ravel()
    rr = np.where(c == 1, r, 3)
    sym = np.stack([v, np.full_like(v, 285), _LSYM[rr], v], 1).ravel()
    exb = np.stack([0 * v, 0 * v, _LEXB[rr], 0 * v], 1).ravel()
    exv = np.stack([0 * v, 0 * v, _LEXV[rr], 0 * v], 1).ravel()
    match = np.stack([0 * v, 1 + 0 * v, 1 + 0 * v, 0 * v], 1).ravel()
    return tuple(np.repeat(x, counts) for x in (sym, exb, exv, match))


def rle_lengths(seq):
    """Code-length sequence -> list of (symbol, extra bits, extra value) with 16 / 17 / 18."""
    out, i = [], 0
    while i < len(seq):
        v, n = seq[i], 1
        while i + n < len(seq) and seq[i + n] == v:
            n += 1
        i += n
        if v == 0:
            while n >= 11:
                k = min(n, 138)
                out.append((18, 7, k - 11))
                n -= k
            if n >= 3:
                out.append((17, 3, n - 3))
                n = 0
            out += [(0, 0, 0)] * n
        else:
            out.append((v, 0, 0))
            n -= 1
            while n >= 3:
                k = min(n, 6)
                out.append((16, 2, k - 3))
                n -= k
            out += [(v, 0, 0)] * n
    return out


def _pack(values, nbits):
    """LSB-first bit packing of (value, width) fields -> bytes (the last byte zero-padded)."""
    values = np.asarray(values, np.int64)
    nbits = np.asarray(nbits, np.int64)
    total = int(nbits.sum())
    idx = np.repeat(np.arange(len(nbits)), nbits)
    within = np.arange(total) - np.repeat(np.cumsum(nbits) - nbits, nbits)
    bits = ((values[idx] >> within) & 1).astype(np.uint8)
    return np.packbits(bits, bitorder="little").tobytes(), total


def dynamic_block(d):
    """(bytes, bit count) of one dynamic block, BFINAL 0, of segment bytes d (without the flush)."""
    sym, exb, exv, match = tokens(d)
    freq = np.bincount(sym, minlength=286).tolist()
    freq[256] = 1
    ll = huffman_lengths(freq, 15)
    lc = canonical_codes(ll)
    nlit = max(257, max(s for s in range(286) if ll[s]) + 1)
    items = rle_lengths(ll[:nlit] + [1])
    clf = [0] * 19
    for s, _, _ in items:
        clf[s] += 1
    cll = huffman_lengths(clf, 7)
    clc = canonical_codes(cll)
    ncl = max(4, max(k for k in range(19) if cll[CL_ORDER[k]]) + 1)
    vals = [4, nlit - 257, 0, ncl - 4] + [cll[CL_ORDER[k]] for k in range(ncl)]
    bits = [3, 5, 5, 4] + [3] * ncl
    for s, eb, ev in items:
        vals.append(clc[s] | (ev << cll[s]))
        bits.append(cll[s] + eb)
    lla, lca = np.asarray(ll, np.int64), np.asarray(lc, np.int64)
    tv = lca[sym] | (exv << lla[sym])                                       # the distance bit of a match is 0
    tb = lla[sym] + exb + match
    vals = np.r_[np.asarray(vals, np.int64), tv, lc[256]]
    bits = np.r_[np.asarray(bits, np.int64), tb, ll[256]]
    return _pack(vals, bits)


def segment_data(d, first):
    """The deflate bytes of one segment (with the zlib header when `first`), full flush included."""
    d = np.asarray(d, np.uint8)
    head = b"\x78\x01" if first else b""
    flush = b"\x00\x00\xff\xff"
    L = len(d)
    stored = b"\x00" + struct.pack("<HH", L, L ^ 0xFFFF) + d.tobytes() + b"\x00" + flush
    dyn, nbits = dynamic_block(d)
    if (nbits + 3 + 7) // 8 + 4 < len(stored):
        # the empty stored block's three zero bits and the padding after the last data bit
        return head + dyn + b"\x00" * ((nbits + 3 + 7) // 8 - len(dyn)) + flush, "dynamic"
    return head + stored, "stored"


def chunk(kind, data):
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data))


def encode(a, return_blocks=False):
    """uint8 [H,W] -> the PNG file the kernels write (bytes); with return_blocks also the block kind per segment."""
    a = np.asarray(a, np.uint8)
    h, w = a.shape
    _, filt = filter_rows(a)
    rows = max(1, SEGMENT_BYTES // (w + 1))
    out = [SIGNATURE, chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 0, 0, 0, 0))]
    kinds = []
    for s, y in enumerate(range(0, h, rows)):
        data, kind = segment_data(filt[y:y + rows].ravel(), s == 0)
        out.append(chunk(b"IDAT", data))
        kinds.append(kind)
    out.append(chunk(b"IDAT", b"\x03\x00" + struct.pack(">I", zlib.adler32(filt.tobytes()))))
    out.append(chunk(b"IEND", b""))
    data = b"".join(out)
    return (data, kinds) if return_blocks else data


def chunks(data):
    """Parse a PNG into [(type, payload, crc ok)] after checking the signature."""
    assert data[:8] == SIGNATURE
    out, p = [], 8
    while p < len(data):
        n = struct.unpack(">I", data[p:p + 4])[0]
        kind, payload = data[p + 4:p + 8], data[p + 8:p + 8 + n]
        crc = struct.unpack(">I", data[p + 8 + n:p + 12 + n])[0]
        out.append((kind, payload, crc == zlib.crc32(kind + payload)))
        p += 12 + n
    return out


def decode(data):
    """Plain decoder: zlib over the concatenated IDAT payloads (which checks the Adler-32), then unfiltering.
    Returns (uint8 [H,W], filter types [H])."""
    cs = chunks(data)
    assert all(ok for _, _, ok in cs)
    w, h, depth, ctype, comp, filt, inter = struct.unpack(">IIBBBBB", cs[0][1])
    assert cs[0][0] == b"IHDR" and (depth, ctype, comp, filt, inter) == (8, 0, 0, 0, 0)
    raw = zlib.decompress(b"".join(p for k, p, _ in cs if k == b"IDAT"))
    rows = np.frombuffer(raw, np.uint8).reshape(h, w + 1)
    out = np.zeros((h, w), np.int32)
    prior = np.zeros(w, np.int32)
    for y in range(h):
        t, f = int(rows[y, 0]), rows[y, 1:].astype(np.int32)
        if t in (0, 2):
            cur = (f + (prior if t == 2 else 0)) & 255
        else:
            cur = np.zeros(w, np.int32)
            for x in range(w):
                a = cur[x - 1] if x else 0
                c = prior[x - 1] if x else 0
                pred = a if t == 1 else (a + prior[x]) // 2 if t == 3 else int(_paeth(np.int32(a), prior[x], np.int32(c)))
                cur[x] = (f[x] + pred) & 255
        out[y] = cur
        prior = cur
    return out.astype(np.uint8), rows[:, 0].copy()
