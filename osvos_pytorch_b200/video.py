"""MJPEG video files from JPEG files (DESIGN.md §25): a RIFF AVI whose frames are the given JPEG files, byte for byte.

``write_avi`` lays out

    RIFF 'AVI '
      LIST 'hdrl'
        avih                   main header: frame period, frame count, one stream, size, AVIF_HASINDEX
        LIST 'strl'
          strh                 'vids' / 'MJPG', rate / scale = the frame rate, length = the frame count
          strf                 BITMAPINFOHEADER, compression 'MJPG', 24 bits
      LIST 'movi'
        00dc ...               one chunk per frame: the JPEG file as given, padded to an even size
      idx1                     per frame: '00dc', AVIIF_KEYFRAME, offset from the 'movi' tag, unpadded size

Nothing is re-encoded, so each frame a player decodes is the JPEG file that was written beside it.  ``read_avi`` walks
the chunks back (the tests use it)."""
import struct
from fractions import Fraction

AVIF_HASINDEX = 0x10
AVIIF_KEYFRAME = 0x10


def jpeg_size(data):
    """(width, height) from a JPEG file's SOF marker."""
    data = bytes(data)
    if data[:2] != b"\xff\xd8":
        raise ValueError("not a JPEG file (no SOI)")
    p = 2
    while p + 4 <= len(data):
        if data[p] != 0xFF:
            raise ValueError("not a JPEG file (marker expected)")
        m = data[p + 1]
        if m == 0xFF:
            p += 1
            continue
        ln, = struct.unpack(">H", data[p + 2:p + 4])
        if 0xC0 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC) and p + 9 <= len(data):
            h, w = struct.unpack(">HH", data[p + 5:p + 9])
            return w, h
        if m == 0xDA:
            break
        p += 2 + ln
    raise ValueError("no SOF marker before the scan")


def _chunk(tag, payload):
    return tag + struct.pack("<I", len(payload)) + payload + (b"\0" if len(payload) % 2 else b"")


def _list(kind, payload):
    return b"LIST" + struct.pack("<I", 4 + len(payload)) + kind + payload


def write_avi(path, frames, fps=24.0):
    """Writes the JPEG files ``frames`` (a list of bytes-like objects of one size) as the MJPEG AVI ``path`` at ``fps``
    frames per second.  Returns the number of bytes written."""
    frames = [bytes(f) for f in frames]
    if not frames:
        raise ValueError("an AVI needs at least one frame")
    rate = Fraction(fps).limit_denominator(1001000)
    if rate <= 0:
        raise ValueError(f"fps must be positive, got {fps}")
    w, h = jpeg_size(frames[0])
    for i, f in enumerate(frames[1:], 1):
        if jpeg_size(f) != (w, h):
            raise ValueError(f"frame {i} is {jpeg_size(f)[0]}x{jpeg_size(f)[1]}, frame 0 {w}x{h}")
    n, biggest = len(frames), max(len(f) for f in frames)
    usec = int(round(1e6 / float(rate)))
    avih = struct.pack("<10I4I", usec, int(biggest * float(rate)) + 1, 0, AVIF_HASINDEX, n, 0, 1, biggest, w, h,
                       0, 0, 0, 0)
    strh = b"vidsMJPG" + struct.pack("<IHHIIIIIIIIhhhh", 0, 0, 0, 0, rate.denominator, rate.numerator, 0, n, biggest,
                                     0xFFFFFFFF, 0, 0, 0, w, h)
    strf = struct.pack("<IiiHH4sIiiII", 40, w, h, 1, 24, b"MJPG", w * h * 3, 0, 0, 0, 0)
    hdrl = _list(b"hdrl", _chunk(b"avih", avih) + _list(b"strl", _chunk(b"strh", strh) + _chunk(b"strf", strf)))
    movi, index, off = [], [], 4                             # idx1 offsets count from the 'movi' tag
    for f in frames:
        c = _chunk(b"00dc", f)
        index.append(struct.pack("<4sIII", b"00dc", AVIIF_KEYFRAME, off, len(f)))
        movi.append(c)
        off += len(c)
    body = b"AVI " + hdrl + _list(b"movi", b"".join(movi)) + _chunk(b"idx1", b"".join(index))
    if len(body) >= 1 << 32:
        raise ValueError("the frames exceed a RIFF file's 4 GiB")
    data = b"RIFF" + struct.pack("<I", len(body)) + body
    with open(path, "wb") as fh:
        fh.write(data)
    return len(data)


def chunks(data, start, end):
    """The chunks of ``data[start:end]``: a list of (tag, payload offset, payload size, list type or None); a LIST's
    payload offset is that of its list type."""
    out = []
    p = start
    while p + 8 <= end:
        tag = data[p:p + 4]
        size, = struct.unpack("<I", data[p + 4:p + 8])
        if p + 8 + size > end:
            raise ValueError(f"chunk {tag!r} at {p} runs past its parent's end")
        out.append((tag, p + 8, size, data[p + 8:p + 12] if tag in (b"LIST", b"RIFF") else None))
        p += 8 + size + (size & 1)
    if p != end:
        raise ValueError(f"{end - p} stray bytes after the last chunk")
    return out


def read_avi(data):
    """An AVI file's bytes -> {'avih', 'strh', 'strf': payload bytes, 'frames': the 00dc payloads in file order,
    'index': the idx1 entries (tag, flags, offset, size), 'movi': the offset of the 'movi' tag}."""
    data = bytes(data)
    (tag, off, size, kind), = chunks(data, 0, len(data))
    if tag != b"RIFF" or kind != b"AVI ":
        raise ValueError("not a RIFF AVI file")
    out = {"frames": []}
    for tag, o, s, kind in chunks(data, off + 4, off + size):
        if kind == b"hdrl":
            for t, o2, s2, k2 in chunks(data, o + 4, o + s):
                if t == b"avih":
                    out["avih"] = data[o2:o2 + s2]
                elif k2 == b"strl":
                    for t3, o3, s3, _ in chunks(data, o2 + 4, o2 + s2):
                        out[t3.decode()] = data[o3:o3 + s3]
        elif kind == b"movi":
            out["movi"] = o
            out["frames"] = [data[o2:o2 + s2] for t, o2, s2, _ in chunks(data, o + 4, o + s) if t == b"00dc"]
        elif tag == b"idx1":
            out["index"] = [struct.unpack("<4sIII", data[o + i:o + i + 16]) for i in range(0, s, 16)]
    return out
