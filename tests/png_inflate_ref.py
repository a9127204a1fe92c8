"""Host restatement of the device PNG decoder's cut verification (csrc/png_decode.cu, png_count_kernel): a plain-Python
raw-deflate reader that inflates one proposed segment on its own and says how many bytes it produces and whether it
is clean.  Slow; for small test files."""

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227,
            258]
LEN_EXTRA = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


class Bad(Exception):
    pass


class Bits:
    def __init__(self, data, beg, end):
        self.data, self.bit, self.end = data, 8 * beg, 8 * end

    def take(self, n):
        if self.bit + n > self.end:
            raise Bad("short")
        v = 0
        for i in range(n):
            v |= ((self.data[(self.bit + i) >> 3] >> ((self.bit + i) & 7)) & 1) << i
        self.bit += n
        return v


def table(lens):
    count = [0] * 16
    for l in lens:
        count[l] += 1
    count[0] = 0
    left = 1
    for l in range(1, 16):
        left = 2 * left - count[l]
        if left < 0:
            raise Bad("over-subscribed")
    if left > 0 and max(lens, default=0) > 1:
        raise Bad("incomplete")
    return count, sorted((s for s, l in enumerate(lens) if l), key=lambda s: (lens[s], s))


def symbol(b, tab):
    count, syms = tab
    code = first = index = 0
    for l in range(1, 16):
        code |= b.take(1)
        if code - count[l] < first:
            return syms[index + code - first]
        index += count[l]
        first = (first + count[l]) << 1
        code <<= 1
    raise Bad("undefined code")


def inflate_segment(data, beg, end, last, limit=1 << 30):
    """Inflates data[beg:end) on its own.  Returns (output bytes, clean): clean as png_count_kernel defines it: no
    error, no distance before the segment's first output byte, and the read position exactly on ``end`` at a block
    boundary (the last segment: BFINAL seen and exactly four bytes left)."""
    b = Bits(data, beg, end)
    out = bytearray()
    try:
        while True:
            final, kind = b.take(1), b.take(2)
            if kind == 0:
                b.bit = (b.bit + 7) & ~7
                n, c = b.take(16), b.take(16)
                if n ^ 0xFFFF != c:
                    raise Bad("stored length")
                if b.bit + 8 * n > b.end:
                    raise Bad("short")
                out += data[b.bit >> 3:(b.bit >> 3) + n]
                b.bit += 8 * n
            elif kind in (1, 2):
                if kind == 1:
                    lit = table([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8)
                    dist = table([5] * 32)
                else:
                    hlit, hdist, hclen = b.take(5) + 257, b.take(5) + 1, b.take(4) + 4
                    if hlit > 286 or hdist > 30:
                        raise Bad("counts")
                    cl = [0] * 19
                    for k in range(hclen):
                        cl[ORDER[k]] = b.take(3)
                    clt = table(cl)
                    lens = []
                    while len(lens) < hlit + hdist:
                        s = symbol(b, clt)
                        if s < 16:
                            lens.append(s)
                        elif s == 16:
                            if not lens:
                                raise Bad("repeat")
                            lens += [lens[-1]] * (3 + b.take(2))
                        elif s == 17:
                            lens += [0] * (3 + b.take(3))
                        else:
                            lens += [0] * (11 + b.take(7))
                    if len(lens) > hlit + hdist or lens[256] == 0:
                        raise Bad("lengths")
                    lit, dist = table(lens[:hlit]), table(lens[hlit:])
                while True:
                    s = symbol(b, lit)
                    if s < 256:
                        out.append(s)
                    elif s == 256:
                        break
                    else:
                        s -= 257
                        if s >= 29:
                            raise Bad("length symbol")
                        n = LEN_BASE[s] + b.take(LEN_EXTRA[s])
                        d = symbol(b, dist)
                        if d >= 30:
                            raise Bad("distance symbol")
                        d = DIST_BASE[d] + b.take(DIST_EXTRA[d])
                        if d > len(out):
                            raise Bad("distance")
                        for _ in range(n):
                            out.append(out[-d])
                    if len(out) > limit:
                        raise Bad("long")
            else:
                raise Bad("block type")
            if final:
                return bytes(out), last and ((b.bit + 7) >> 3) + 4 == end
            if not last and b.bit == b.end:
                return bytes(out), True
    except Bad:
        return bytes(out), False
