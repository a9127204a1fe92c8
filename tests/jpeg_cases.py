"""Seeded JPEG files for the decoder tests: cv2-encoded over sampling, quality, optimised tables, restart intervals,
grayscale and sizes, Pillow-encoded files, a file whose scan is cut short, and files outside the device subset."""
import io
import struct

import numpy as np

SAMPLING = {"444": 0x111111, "422": 0x211111, "440": 0x121111, "420": 0x221111}
SIZES = [(1, 1), (1, 17), (8, 8), (16, 16), (33, 45), (48, 70), (97, 131)]


def picture(h, w, seed=0, saturated=False):
    """A frame with gradients, texture and edges (uint8 BGR); ``saturated``: large flat areas at 0 and 255 with hard
    edges, where quality 100 pushes the IDCT past the 8-bit range."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[:h, :w]
    a = np.stack([x * 255 // max(w - 1, 1), y * 255 // max(h - 1, 1), ((x + y) * 7) % 256], -1).astype(np.int32)
    a += rng.integers(-40, 40, a.shape)
    if saturated:
        a = np.where(((x // 3 + y // 5) % 2)[..., None] == 0, 255, 0) * np.array([1, 0, 1]) + \
            np.where((x + y) % 4 < 2, 255, 0)[..., None] * np.array([0, 1, 0])
    return np.clip(a, 0, 255).astype(np.uint8)


def cv2_file(img, quality=75, sampling="420", optimize=False, restart=0, gray=False):
    import cv2
    params = [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLING[sampling],
              cv2.IMWRITE_JPEG_OPTIMIZE, int(optimize), cv2.IMWRITE_JPEG_RST_INTERVAL, restart]
    if gray:
        img = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
    ok, buf = cv2.imencode(".jpg", img, params)
    assert ok
    return buf.tobytes()


def cv2_matrix():
    """name -> file bytes over the cv2 encoder's options."""
    out = {}
    for s in SAMPLING:
        for (h, w) in SIZES:
            for q in (5, 50, 75, 95, 100):
                out[f"cv2_{s}_q{q}_{h}x{w}"] = cv2_file(picture(h, w, seed=h * 1000 + w), q, s)
        out[f"cv2_{s}_q100_sat"] = cv2_file(picture(64, 80, saturated=True), 100, s)
        out[f"cv2_{s}_opt"] = cv2_file(picture(97, 131, seed=3), 85, s, optimize=True)
        for r in (1, 7):
            out[f"cv2_{s}_rst{r}"] = cv2_file(picture(97, 131, seed=4), 80, s, restart=r)
        mcu_row = -(-131 // (16 if s in ("420", "422") else 8))
        out[f"cv2_{s}_rstrow"] = cv2_file(picture(97, 131, seed=5), 80, s, restart=mcu_row)
    for (h, w) in SIZES + [(480, 854)]:
        out[f"cv2_gray_{h}x{w}"] = cv2_file(picture(h, w, seed=7), 80, gray=True)
    out["cv2_gray_rst7"] = cv2_file(picture(97, 131, seed=8), 80, gray=True, restart=7)
    out["cv2_420_q75_480x854"] = cv2_file(picture(480, 854, seed=9), 75, "420")
    out["cv2_420_q95_480x854"] = cv2_file(picture(480, 854, seed=9), 95, "420")
    return out


def pillow_files():
    from PIL import Image
    out = {}
    for sub, name in ((0, "444"), (1, "422"), (2, "420")):
        for q in (30, 90):
            img = Image.fromarray(picture(61, 83, seed=11)[..., ::-1].copy())
            buf = io.BytesIO()
            img.save(buf, "JPEG", quality=q, subsampling=sub)
            out[f"pil_{name}_q{q}"] = buf.getvalue()
    buf = io.BytesIO()
    Image.fromarray(picture(50, 60, seed=12)[..., 0].copy()).save(buf, "JPEG", quality=70)
    out["pil_gray"] = buf.getvalue()
    return out


def cut_short(buf, keep=0.6):
    """The file with its scan cut after ``keep`` of the entropy-coded bytes and EOI appended."""
    sos = buf.index(b"\xff\xda")
    body = sos + 2 + ((buf[sos + 2] << 8) | buf[sos + 3])
    end = body + int((len(buf) - 2 - body) * keep)
    if buf[end - 1] == 0xFF:
        end -= 1
    return buf[:end] + b"\xff\xd9"


def with_app(buf, marker, payload):
    """``buf`` with an APPn segment inserted after SOI (replacing a JFIF APP0 when inserting APP14)."""
    body = buf[2:]
    if marker == 0xEE and body[:2] == b"\xff\xe0":
        body = body[2 + ((body[2] << 8) | body[3]):]
    return b"\xff\xd8" + bytes([0xFF, marker]) + struct.pack(">H", len(payload) + 2) + payload + body


def exif(orientation):
    tiff = b"II*\x00" + struct.pack("<I", 8) + struct.pack("<H", 1) + struct.pack("<HHII", 0x0112, 3, 1, orientation) \
        + struct.pack("<I", 0)
    return b"Exif\x00\x00" + tiff


def adobe(transform):
    return b"Adobe" + struct.pack(">HHHB", 100, 0, 0, transform)


def patch_sof(buf, new_marker=None, precision=None):
    i = buf.index(b"\xff\xc0")
    b = bytearray(buf)
    if new_marker is not None:
        b[i + 1] = new_marker
    if precision is not None:
        b[i + 4] = precision
    return bytes(b)


def fallback_files():
    """name -> (file bytes, expected reason fragment)."""
    import cv2
    img = picture(48, 70, seed=13)
    base = cv2_file(img, 75, "420")
    ok, prog = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])
    ok, s411 = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x411111])
    return {
        "progressive": (prog.tobytes(), "progressive"),
        "411": (s411.tobytes(), "sampling"),
        "exif6": (with_app(base, 0xE1, exif(6)), "EXIF"),
        "adobe0": (with_app(base, 0xEE, adobe(0)), "RGB"),
        "sof9": (patch_sof(base, new_marker=0xC9), "arithmetic"),
        "sof3": (patch_sof(base, new_marker=0xC3), "lossless"),
        "12bit": (patch_sof(base, precision=12), "precision"),
        "truncated": (base[:base.index(b"\xff\xc4") + 10], "truncated"),
        "no_sos": (base[:base.index(b"\xff\xda")] + b"\xff\xd9", "SOS"),
    }
