"""numpy restatement of libjpeg-turbo's baseline compression as cv2.imencode('.jpg', frame, [IMWRITE_JPEG_QUALITY, q])
configures it: 4:2:0, ISLOW FDCT, the Annex K Huffman tables, no restart interval (DESIGN.md §23).  The oracle of
tests/test_jpeg_encode.py and the model csrc/jpeg_encode.cu restates:

  colour     jccolor.c rgb_ycc_convert, 16 fractional bits;
  edges      jcprepct.c / jcsample.c: columns replicated to whole MCUs (16) before the chroma downsampling, rows to an
             even count; after downsampling every plane's rows are replicated to the whole iMCU row;
  chroma     jcsample.c h2v2_downsample: (sum of 2x2 + bias) >> 2, bias 1, 2, 1, 2, ... along each output row;
  FDCT       jfdctint.c jpeg_fdct_islow on samples - 128;
  quantise   jcdctmgr.c: |x| * 2^r / (8 q) by libjpeg-turbo's reciprocal, sign restored (equal to round half away
             from zero, ``quant_divide`` checks it over the whole domain);
  dummies    jccoefct.c compress_data: luma blocks of the last MCU column / row outside the image have AC 0 and the DC of
             the block to their left (right edge: blocks 1 and 3 from 0 and 2) or of block 1 (bottom edge: blocks 2
             and 3, after block 1's own right-edge copy);
  entropy    jchuff.c with the standard tables, DC predicted per component over the whole scan, FF -> FF 00, the last
             byte padded with 1 bits."""
import numpy as np

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                   6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45,
                   38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])

STD_LUMA_Q = np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                       14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113,
                       92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99])
STD_CHROMA_Q = np.array([17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
                         47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32)

# Annex K.3: (counts of codes of length 1..16, symbols)
DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D], [
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07,
    0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xA1, 0x08, 0x23, 0x42, 0xB1, 0xC1, 0x15, 0x52, 0xD1, 0xF0,
    0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0A, 0x16, 0x17, 0x18, 0x19, 0x1A, 0x25, 0x26, 0x27, 0x28,
    0x29, 0x2A, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49,
    0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89,
    0x8A, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7,
    0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3, 0xC4, 0xC5,
    0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8, 0xD9, 0xDA, 0xE1, 0xE2,
    0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF1, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8,
    0xF9, 0xFA])
AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], [
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71,
    0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xA1, 0xB1, 0xC1, 0x09, 0x23, 0x33, 0x52, 0xF0,
    0x15, 0x62, 0x72, 0xD1, 0x0A, 0x16, 0x24, 0x34, 0xE1, 0x25, 0xF1, 0x17, 0x18, 0x19, 0x1A, 0x26,
    0x27, 0x28, 0x29, 0x2A, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
    0x69, 0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87,
    0x88, 0x89, 0x8A, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5,
    0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3,
    0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8, 0xD9, 0xDA,
    0xE2, 0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8,
    0xF9, 0xFA])

HEADER_BYTES = 623
BLOCK_BITS_MAX = 22 + 63 * 26        # DC: 11-bit code + 11 bits; 63 AC of a 16-bit code + 10 bits each


def max_bytes(h, w):
    """The per-file capacity osvos_jpeg_max_bytes gives: every block at its largest, every byte stuffed."""
    units = 6 * (-(-h // 16)) * (-(-w // 16))
    return HEADER_BYTES + 2 + 2 * (-(-units * BLOCK_BITS_MAX // 8))


def quant_table(base, quality):
    """jcparam.c jpeg_set_quality -> jpeg_add_quant_table with force_baseline."""
    q = min(max(int(quality), 1), 100)
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return np.clip((base * scale + 50) // 100, 1, 255).astype(np.int64)


def quant_divide(x, div):
    """jcdctmgr.c quantize with compute_reciprocal's (reciprocal, correction, shift) for the divisor 8 q."""
    div = np.asarray(div, np.int64)
    b = np.floor(np.log2(div)).astype(np.int64)
    r = 16 + b
    fq = (np.int64(1) << r) // div
    fr = (np.int64(1) << r) % div
    c = div // 2
    pow2 = fr == 0
    fq = np.where(pow2, fq >> 1, np.where(fr <= div // 2, fq, fq + 1))
    c = np.where(pow2, c, np.where(fr <= div // 2, c + 1, c))
    r = np.where(pow2, r - 1, r)
    a = np.abs(x)
    v = ((a + c) * fq) >> r
    return np.where(x < 0, -v, v)


def huff_codes(spec):
    """Canonical codes of a (counts, symbols) table -> (code[256], size[256])."""
    counts, syms = spec
    code = np.zeros(256, np.int64)
    size = np.zeros(256, np.int64)
    c, k = 0, 0
    for length in range(1, 17):
        for _ in range(counts[length - 1]):
            code[syms[k]], size[syms[k]] = c, length
            c += 1
            k += 1
        c <<= 1
    return code, size


def header(h, w, quality):
    """SOI, JFIF APP0, two DQT, SOF0 (4:2:0), four DHT, SOS: 623 bytes that depend on (h, w, quality) alone."""
    out = bytearray(b"\xFF\xD8\xFF\xE0\x00\x10JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for t, base in enumerate((STD_LUMA_Q, STD_CHROMA_Q)):
        out += bytes([0xFF, 0xDB, 0, 67, t]) + bytes(int(v) for v in quant_table(base, quality)[ZIGZAG])
    out += bytes([0xFF, 0xC0, 0, 17, 8, h >> 8, h & 255, w >> 8, w & 255, 3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1])
    for cls_id, spec in ((0x00, DC_LUMA), (0x10, AC_LUMA), (0x01, DC_CHROMA), (0x11, AC_CHROMA)):
        counts, syms = spec
        n = 19 + len(syms)
        out += bytes([0xFF, 0xC4, n >> 8, n & 255, cls_id] + counts + syms)
    out += bytes([0xFF, 0xDA, 0, 12, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0])
    assert len(out) == HEADER_BYTES
    return bytes(out)


def _fix16(x):
    return int(x * 65536 + 0.5)


def ycc(frame):
    """BGR uint8 [H][W][3] -> (Y, Cb, Cr) int64 planes, jccolor.c."""
    b, g, r = (frame[..., i].astype(np.int64) for i in range(3))
    half = 1 << 15
    y = (_fix16(0.299) * r + _fix16(0.587) * g + _fix16(0.114) * b + half) >> 16
    cb = (-_fix16(0.16874) * r - _fix16(0.33126) * g + _fix16(0.5) * b + (128 << 16) + half - 1) >> 16
    cr = (_fix16(0.5) * r - _fix16(0.41869) * g - _fix16(0.08131) * b + (128 << 16) + half - 1) >> 16
    return y, cb, cr


def planes(frame):
    """-> Y [16 my][16 mx] and Cb, Cr [8 my][8 mx] int64, edges replicated as jcprepct.c / jcsample.c do."""
    h, w = frame.shape[:2]
    my, mx = -(-h // 16), -(-w // 16)
    y, cb, cr = ycc(frame)
    ys = y[np.minimum(np.arange(16 * my), h - 1)][:, np.minimum(np.arange(16 * mx), w - 1)]
    ch = []
    hr = h + (h & 1)
    for p in (cb, cr):
        e = p[np.minimum(np.arange(hr), h - 1)][:, np.minimum(np.arange(16 * mx), w - 1)]
        s = e[0::2, 0::2] + e[0::2, 1::2] + e[1::2, 0::2] + e[1::2, 1::2]
        bias = np.where(np.arange(8 * mx) & 1, 2, 1)
        d = (s + bias) >> 2                                          # ceil(h / 2) rows
        ch.append(d[np.minimum(np.arange(8 * my), d.shape[0] - 1)])
    return ys, ch[0], ch[1]


def fdct_islow(blocks):
    """jpeg_fdct_islow on int [B][8][8] (samples - 128) -> int [B][8][8], scaled by 8."""
    def pass_(d, final):
        t0, t7 = d[0] + d[7], d[0] - d[7]
        t1, t6 = d[1] + d[6], d[1] - d[6]
        t2, t5 = d[2] + d[5], d[2] - d[5]
        t3, t4 = d[3] + d[4], d[3] - d[4]
        t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
        sh = 13 + 2 if final else 13 - 2
        ds = lambda v, n=sh: (v + (1 << (n - 1))) >> n
        o = [None] * 8
        if final:
            o[0], o[4] = ds(t10 + t11, 2), ds(t10 - t11, 2)
        else:
            o[0], o[4] = (t10 + t11) << 2, (t10 - t11) << 2
        z1 = (t12 + t13) * 4433
        o[2] = ds(z1 + t13 * 6270)
        o[6] = ds(z1 - t12 * 15137)
        z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
        z5 = (z3 + z4) * 9633
        t4, t5, t6, t7 = t4 * 2446, t5 * 16819, t6 * 25172, t7 * 12299
        z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069 + z5, z4 * -3196 + z5
        o[7] = ds(t4 + z1 + z3)
        o[5] = ds(t5 + z2 + z4)
        o[3] = ds(t6 + z2 + z3)
        o[1] = ds(t7 + z1 + z4)
        return o
    rows = pass_([blocks[:, :, i] for i in range(8)], False)       # over each row: index = column
    ws = np.stack(rows, axis=2)                                     # [B][row][u]
    cols = pass_([ws[:, i, :] for i in range(8)], True)            # over each column
    return np.stack(cols, axis=1)                                   # [B][v][u]


def _blocks(plane):
    hb, wb = plane.shape[0] // 8, plane.shape[1] // 8
    return plane.reshape(hb, 8, wb, 8).transpose(0, 2, 1, 3).reshape(hb, wb, 8, 8)


def coefficients(frame, quality):
    """-> int64 [MCUs * 6][64] quantised coefficients in zig-zag order, MCU interleave order (Y0 Y1 Y2 Y3 Cb Cr),
    dummy blocks included."""
    h, w = frame.shape[:2]
    my, mx = -(-h // 16), -(-w // 16)
    ys, cb, cr = planes(frame)
    qy, qc = quant_table(STD_LUMA_Q, quality), quant_table(STD_CHROMA_Q, quality)
    out = []
    for plane, q in ((ys, qy), (cb, qc), (cr, qc)):
        b = _blocks(plane)
        hb, wb = b.shape[:2]
        d = fdct_islow(b.reshape(-1, 8, 8) - 128).reshape(hb * wb, 64)
        out.append(quant_divide(d, 8 * q)[:, ZIGZAG].reshape(hb, wb, 64))
    y = out[0].reshape(my, 2, mx, 2, 64).transpose(0, 2, 1, 3, 4).reshape(my, mx, 4, 64).copy()
    hib, wib = -(-h // 8), -(-w // 8)
    if wib & 1:                                                     # right dummies: blocks 1, 3 from blocks 0, 2
        y[:, -1, 1::2] = 0
        y[:, -1, 1::2, 0] = y[:, -1, 0::2, 0]
    if hib & 1:                                                     # bottom dummies: blocks 2, 3 from block 1
        y[-1, :, 2:] = 0
        y[-1, :, 2:, 0] = y[-1, :, 1:2, 0]
    mcu = np.concatenate([y, out[1][:, :, None], out[2][:, :, None]], axis=2)
    return mcu.reshape(my * mx * 6, 64)


def entropy(coef):
    """jchuff.c encode_one_block over [MCUs * 6][64] zig-zag coefficients -> the scan's bytes, stuffed and padded."""
    nb = coef.shape[0]
    comp = np.tile(np.array([0, 0, 0, 0, 1, 2]), nb // 6)
    tabs = [(huff_codes(DC_LUMA), huff_codes(AC_LUMA)), (huff_codes(DC_CHROMA), huff_codes(AC_CHROMA))]
    tab = np.minimum(comp, 1)
    dc = coef[:, 0]
    prev = np.zeros(nb, np.int64)
    for c in range(3):
        idx = np.nonzero(comp == c)[0]
        prev[idx[1:]] = dc[idx[:-1]]
    keys, vals, lens = [], [], []

    def nbits(a):
        a = np.abs(a)
        return np.where(a > 0, np.floor(np.log2(np.maximum(a, 1))).astype(np.int64) + 1, 0)

    def extra(v, s):
        return np.where(v < 0, v - 1, v) & ((np.int64(1) << s) - 1)

    diff = dc - prev
    s = nbits(diff)
    code = np.where(tab == 0, tabs[0][0][0][s], tabs[1][0][0][s])
    size = np.where(tab == 0, tabs[0][0][1][s], tabs[1][0][1][s])
    keys.append(np.arange(nb) * 256)
    vals.append((code << s) | extra(diff, s))
    lens.append(size + s)
    bi, k = np.nonzero(coef[:, 1:])
    k = k + 1
    v = coef[bi, k]
    first = np.ones(len(bi), bool)
    first[1:] = bi[1:] != bi[:-1]
    prevk = np.where(first, 0, np.concatenate([[0], k[:-1]]))
    run = k - prevk - 1
    zrl = run >> 4
    run = run & 15
    s = nbits(v)
    sym = (run << 4) | s
    t = tab[bi]
    code = np.where(t == 0, tabs[0][1][0][sym], tabs[1][1][0][sym])
    size = np.where(t == 0, tabs[0][1][1][sym], tabs[1][1][1][sym])
    zc = np.where(t == 0, tabs[0][1][0][0xF0], tabs[1][1][0][0xF0])
    zs = np.where(t == 0, tabs[0][1][1][0xF0], tabs[1][1][1][0xF0])
    for j in range(3):                                              # up to 3 ZRLs before a coefficient
        m = zrl > j
        keys.append(bi[m] * 256 + 2 * k[m] - 1)
        vals.append(zc[m])
        lens.append(zs[m])
    keys.append(bi * 256 + 2 * k)
    vals.append((code << s) | extra(v, s))
    lens.append(size + s)
    last = np.full(nb, 0)
    np.maximum.at(last, bi, k)
    e = np.nonzero(last < 63)[0]
    keys.append(e * 256 + 200)
    vals.append(np.where(tab[e] == 0, tabs[0][1][0][0], tabs[1][1][0][0]))
    lens.append(np.where(tab[e] == 0, tabs[0][1][1][0], tabs[1][1][1][0]))
    keys, vals, lens = (np.concatenate(a) for a in (keys, vals, lens))
    order = np.argsort(keys, kind="stable")
    vals, lens = vals[order], lens[order]
    total = int(lens.sum())
    start = np.cumsum(lens) - lens
    ent = np.repeat(np.arange(len(lens)), lens)
    off = np.arange(total) - start[ent]
    bits = (vals[ent] >> (lens[ent] - 1 - off)) & 1
    bits = np.concatenate([bits, np.ones((-total) % 8, np.int64)]).astype(np.uint8)
    data = np.packbits(bits)
    ff = np.nonzero(data == 0xFF)[0]
    return np.insert(data, ff + 1, 0).tobytes()


def encode(frame, quality=95):
    """uint8 BGR [H][W][3] -> the JPEG file cv2.imencode('.jpg', frame, [cv2.IMWRITE_JPEG_QUALITY, quality]) writes."""
    frame = np.ascontiguousarray(frame, np.uint8)
    h, w = frame.shape[:2]
    return header(h, w, quality) + entropy(coefficients(frame, quality)) + b"\xFF\xD9"
