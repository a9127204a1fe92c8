"""Python restatement of libjpeg-turbo's baseline decode as cv2.imread configures it, over jpeg.parse's output: the
Huffman decoder (jdhuff.c, with zero bits past a segment's end and the rest of an early-ended segment left zero),
ISLOW IDCT (jidctint.c), fancy upsampling (jdsample.c) and YCbCr -> BGR (jdcolor.c).  The oracle of tests/test_jpeg.py
and the model csrc/jpeg.cu restates; the chunked synchronising decode (``decode_chunked``) is the kernel's algorithm.

Decoder state at a symbol boundary: (bit position in the segment, block within the MCU, zig-zag index)."""
import numpy as np

from osvos_pytorch_b200.jpeg import LOOKAHEAD, ZIGZAG

NATURAL = np.concatenate([ZIGZAG, np.full(16, 63, np.int32)])     # jpeg_natural_order with its 16 guard entries


class Segment:
    def __init__(self, data):
        self.nbits = 8 * len(data)
        self.d = bytes(data) + b"\0" * 8

    def peek16(self, pos):
        if pos >= self.nbits:
            return 0
        b = pos >> 3
        v = ((self.d[b] << 16) | (self.d[b + 1] << 8) | self.d[b + 2]) >> (8 - (pos & 7)) & 0xFFFF
        rem = self.nbits - pos                        # bits past the end read as zero
        return v if rem >= 16 else v & ~((1 << (16 - rem)) - 1) & 0xFFFF

    def bits(self, pos, n):
        return self.peek16(pos) >> (16 - n) if n else 0


def huff_decode(seg, pos, t):
    """-> (symbol, code length); a bad code decodes as symbol 0 after 16 bits (bad=True)."""
    v = seg.peek16(pos)
    e = int(t.lookup[v >> (16 - LOOKAHEAD)])
    if (e >> 8) <= LOOKAHEAD:
        return e & 0xFF, e >> 8, False
    for l in range(LOOKAHEAD + 1, 17):
        code = v >> (16 - l)
        if code <= t.maxcode[l]:
            return int(t.vals[(code + t.valoffset[l]) & 0xFF]), l, False
    return 0, 16, True


def extend(r, s):
    return r - (1 << s) + 1 if r < (1 << (s - 1)) else r


def block_components(p):
    return [0] * (p.hs * p.vs) + [1, 2] if p.ncomp == 3 else [0]


def decode_span(p, seg, state, end, last, emit=None):
    """Decode from ``state`` while pos < end (``last``: the segment's last chunk, which stops only at an MCU boundary
    past the segment's end, libjpeg's insufficient-data rule).  ``emit(block, zz, value, bad)`` receives every
    coefficient (zz 0: the DC difference) and emit(block, -1, end_pos, flags) at each block's end, with ``block`` the
    count of blocks completed so far in this span.  -> (exit state, blocks completed)."""
    comps = block_components(p)
    bpm = len(comps)
    pos, blk, zz = state
    nblocks = 0
    flags = 0
    while True:
        if last:
            if blk == 0 and zz == 0 and pos > seg.nbits:
                break
        elif pos >= end:
            break
        c = comps[blk]
        if zz == 0:
            s, l, bad = huff_decode(seg, pos, p.dc[c])
            flags |= bad
            pos += l
            v = extend(seg.bits(pos, s), s) if s else 0
            pos += s
            if emit:
                emit(nblocks, 0, v, 0)
            zz = 1
        else:
            rs, l, bad = huff_decode(seg, pos, p.ac[c])
            flags |= bad
            pos += l
            r, s = rs >> 4, rs & 15
            if s:
                zz += r
                if zz > 63:
                    flags |= 2
                v = extend(seg.bits(pos, s), s)
                pos += s
                if emit:
                    emit(nblocks, zz, v, 0)
                zz += 1
            elif r == 15:
                zz += 16
                if zz > 64:
                    flags |= 2
            else:
                zz = 64
        if zz >= 64:
            if emit:
                emit(nblocks, -1, pos, flags)
            flags = 0
            nblocks += 1
            zz = 0
            blk = blk + 1 if blk + 1 < bpm else 0
    return (pos, blk, zz), nblocks


def _writer(coef, first, limit, status, seg):
    """An emit callback writing one segment's coefficients (natural order) from block ``first`` on, capped at
    ``limit`` blocks; status bits: 1 bad Huffman code, 2 zig-zag index past 63, 4 data ended before the last MCU."""
    def emit(b, zz, v, flags):
        if b >= limit:
            return
        if zz < 0:
            status[0] |= flags & 3
            if v > seg.nbits:
                status[0] |= 4
            return
        coef[first + b, NATURAL[min(zz, 79)]] = v
    return emit


def coefficients(p, chunk_bits=None):
    """Quantised coefficients int32 [blocks][64] in natural order (DC absolute) and the status word.  chunk_bits None:
    one sequential decode per segment; otherwise decode_chunked's synchronised chunks."""
    bpm = p.bpm
    total = p.mcux * p.mcuy * bpm
    per = (p.restart or p.mcux * p.mcuy) * bpm
    coef = np.zeros((total, 64), np.int64)
    status = [0]
    comps = np.array(block_components(p) * (total // bpm))
    for si, data in enumerate(p.segments):
        seg = Segment(data)
        first = si * per
        limit = min(per, total - first)
        if chunk_bits is None:
            _, done = decode_span(p, seg, (0, 0, 0), seg.nbits, True, _writer(coef, first, limit, status, seg))
        else:
            done = decode_chunked(p, seg, chunk_bits, _writer(coef, first, limit, status, seg))
        done = min(done, limit)
        if done < limit:
            status[0] |= 4
        for c in range(p.ncomp):                      # DC: running sum per component, reset at each restart
            idx = np.flatnonzero(comps[first:first + done] == c) + first
            coef[idx, 0] = np.cumsum(coef[idx, 0])
        coef[first + done:first + limit] = 0          # libjpeg leaves MCUs after the data ran out all zero
    return coef, status[0]


def decode_chunked(p, seg, S, emit):
    """The kernel's algorithm on one segment: chunks of S bits decoded speculatively from (chunk start, 0, 0), then
    re-decoded in rounds from the predecessor's exit state until no exit changes; block offsets by a prefix sum of
    the chunk counts; then each chunk writes from its synced entry.  -> blocks decoded."""
    nch = max(1, -(-seg.nbits // S))
    ends = [min((c + 1) * S, seg.nbits) for c in range(nch)]
    entry = [(c * S, 0, 0) for c in range(nch)]
    res = [decode_span(p, seg, entry[c], ends[c], c == nch - 1) for c in range(nch)]
    rounds = 0
    while True:
        changed = False
        new = list(res)
        for c in range(1, nch):
            if res[c - 1][0] != entry[c]:
                entry[c] = res[c - 1][0]
                new[c] = decode_span(p, seg, entry[c], ends[c], c == nch - 1)
                changed = True
        res = new
        rounds += 1
        assert rounds <= nch
        if not changed:
            break
    first = np.concatenate([[0], np.cumsum([r[1] for r in res])])
    for c in range(nch):
        decode_span(p, seg, entry[c], ends[c], c == nch - 1,
                    lambda b, zz, v, f, o=int(first[c]): emit(o + b, zz, v, f))
    return int(first[-1])


# ---- pixels ------------------------------------------------------------------------------------------------------
C13 = {k: v for k, v in dict(c0298=2446, c0390=3196, c0541=4433, c0765=6270, c0899=7373, c1175=9633, c1501=12299,
                             c1847=15137, c1961=16069, c2053=16819, c2562=20995, c3072=25172).items()}


def _idct_1d(x0, x1, x2, x3, x4, x5, x6, x7, k):
    z1 = (x2 + x6) * C13["c0541"]
    tmp2 = z1 - x6 * C13["c1847"]
    tmp3 = z1 + x2 * C13["c0765"]
    tmp0 = (x0 + x4) << 13
    tmp1 = (x0 - x4) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    a0, a1, a2, a3 = x7, x5, x3, x1
    z1, z2, z3, z4 = a0 + a3, a1 + a2, a0 + a2, a1 + a3
    z5 = (z3 + z4) * C13["c1175"]
    a0, a1, a2, a3 = a0 * C13["c0298"], a1 * C13["c2053"], a2 * C13["c3072"], a3 * C13["c1501"]
    z1, z2 = z1 * -C13["c0899"], z2 * -C13["c2562"]
    z3, z4 = z3 * -C13["c1961"] + z5, z4 * -C13["c0390"] + z5
    a0, a1, a2, a3 = a0 + z1 + z3, a1 + z2 + z4, a2 + z2 + z3, a3 + z1 + z4
    r = 1 << (k - 1)
    return [(t10 + a3 + r) >> k, (t11 + a2 + r) >> k, (t12 + a1 + r) >> k, (t13 + a0 + r) >> k,
            (t13 - a0 + r) >> k, (t12 - a1 + r) >> k, (t11 - a2 + r) >> k, (t10 - a3 + r) >> k]


def idct_islow(coef, q):
    """jpeg_idct_islow on [B][64] natural-order coefficients (int64) with quant table q [64] -> uint8 [B][8][8]."""
    d = (coef * q.astype(np.int64)).reshape(-1, 8, 8)            # [B][row v][col u]
    cols = _idct_1d(*[d[:, i, :] for i in range(8)], 11)          # pass 1 over columns: rows 0..7 of [B][u]
    ws = np.stack(cols, axis=1)                                   # [B][y][u]
    rows = _idct_1d(*[ws[:, :, i] for i in range(8)], 18)         # pass 2 over rows
    out = np.stack(rows, axis=2)                                  # [B][y][x]
    s = ((out & 1023) ^ 512) - 512                                # the 10-bit range-limit wrap, then clamp
    return np.clip(s + 128, 0, 255).astype(np.uint8)


def planes(p, coef):
    """Component planes uint8, each padded to whole MCUs."""
    comps = block_components(p)
    bpm = len(comps)
    out = []
    for c in range(p.ncomp):
        hs, vs = (p.hs, p.vs) if c == 0 else (1, 1)
        ks = [k for k in range(bpm) if comps[k] == c]
        pix = idct_islow(coef[[m * bpm + k for m in range(p.mcux * p.mcuy) for k in ks]], p.qt[c])
        pix = pix.reshape(p.mcuy, p.mcux, vs, hs, 8, 8).transpose(0, 2, 4, 1, 3, 5)
        out.append(pix.reshape(p.mcuy * vs * 8, p.mcux * hs * 8))
    return out


def _h2(row, dw):
    """h2v1 fancy upsampling of int rows [..., dw] -> [..., 2 dw]."""
    r = row.astype(np.int64)
    if dw <= 2:
        return np.repeat(r, 2, axis=-1)
    left = np.concatenate([r[..., :1], (3 * r[..., 1:] + r[..., :-1] + 1) >> 2], axis=-1)
    right = np.concatenate([(3 * r[..., :-1] + r[..., 1:] + 2) >> 2, r[..., -1:]], axis=-1)
    left[..., 0] = r[..., 0]
    return np.stack([left, right], axis=-1).reshape(*r.shape[:-1], 2 * dw)


def upsample(p, plane):
    """A chroma plane at the luma resolution (libjpeg-turbo's fancy upsampling and its edge rules) -> int [H][W]."""
    h, w = p.h, p.w
    dw, dh = -(-w // p.hs), -(-h // p.vs)
    c = plane[:dh, :dw].astype(np.int64)
    if p.hs == 1 and p.vs == 1:
        return c
    if p.vs == 1:
        return _h2(c, dw)[:, :w]
    y = np.arange(h)
    r = y >> 1
    r1 = np.clip(np.where(y & 1, r + 1, r - 1), 0, dh - 1)
    if p.hs == 1:                                                 # h1v2
        return (3 * c[r] + c[r1] + np.where(y & 1, 2, 1)[:, None]) >> 2
    if dw <= 2:                                                   # h2v2 box
        return np.repeat(c[r], 2, axis=1)[:, :w]
    cs = 3 * c[r] + c[r1]                                         # column sums [H][dw]
    even = np.concatenate([(cs[:, :1] * 4 + 8) >> 4, (3 * cs[:, 1:] + cs[:, :-1] + 8) >> 4], axis=1)
    odd = np.concatenate([(3 * cs[:, :-1] + cs[:, 1:] + 7) >> 4, (cs[:, -1:] * 4 + 7) >> 4], axis=1)
    return np.stack([even, odd], axis=-1).reshape(h, 2 * dw)[:, :w]


def _fix(x):
    return int(x * 65536 + 0.5)


def ycc_to_bgr(y, cb, cr):
    """jdcolor.c's ycc_rgb_convert (16 fractional bits) -> uint8 [H][W][3] BGR."""
    y, cb, cr = (np.asarray(v, np.int64) for v in (y, cb, cr))
    xb, xr = cb - 128, cr - 128
    half = 1 << 15
    r = y + ((_fix(1.40200) * xr + half) >> 16)
    b = y + ((_fix(1.77200) * xb + half) >> 16)
    g = y + ((-_fix(0.34414) * xb + half - _fix(0.71414) * xr) >> 16)
    return np.clip(np.stack([b, g, r], axis=-1), 0, 255).astype(np.uint8)


def decode(p, chunk_bits=None):
    """Parsed -> (uint8 [H][W][3] BGR as cv2.imread gives it, status word)."""
    coef, status = coefficients(p, chunk_bits)
    pl = planes(p, coef)
    y = pl[0][:p.h, :p.w]
    if p.ncomp == 1:
        return np.repeat(y[:, :, None], 3, axis=2), status
    return ycc_to_bgr(y, upsample(p, pl[1]), upsample(p, pl[2])), status
