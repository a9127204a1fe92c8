"""The numpy restatement of the JPEG encoder (tests/jpeg_encode_ref.py) against cv2.imencode, byte for byte, and its
files against the project's parser and decoder restatement."""
import os

import numpy as np
import pytest

import jpeg_encode_cases as C
import jpeg_encode_ref as R
import jpeg_ref
from osvos_pytorch_b200 import jpeg

cv2 = pytest.importorskip("cv2")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_jpeg_encode.npz")


def _cv2(frame, q):
    ok, buf = cv2.imencode(".jpg", frame, [cv2.IMWRITE_JPEG_QUALITY, q])
    assert ok
    return buf.tobytes()


@pytest.mark.parametrize("h,w", C.SIZES)
def test_restatement_equals_cv2(h, w):
    for kind in C.KINDS:
        f = C.frame(h, w, kind)
        for q in C.QUALITIES:
            got = R.encode(f, q)
            assert got == _cv2(f, q), (h, w, kind, q)
            assert len(got) <= R.max_bytes(h, w)


@pytest.mark.parametrize("h,w", [(7, 9), (17, 33), (97, 131), (480, 854)])
def test_files_parse_and_decode_as_cv2_decodes_them(h, w):
    for kind in ("noise", "overlay"):
        f = C.frame(h, w, kind)
        for q in (5, 95, 100):
            buf = R.encode(f, q)
            p = jpeg.parse(buf)
            assert isinstance(p, jpeg.Parsed), (h, w, kind, q, p)
            got, status = jpeg_ref.decode(p)
            assert status == 0
            assert np.array_equal(got, cv2.imdecode(np.frombuffer(buf, np.uint8), cv2.IMREAD_COLOR))


def test_header_depends_on_size_and_quality_only():
    for q in C.QUALITIES:
        for h, w in [(1, 1), (480, 854), (65500, 65500)]:
            hd = R.header(h, w, q)
            assert len(hd) == R.HEADER_BYTES
        assert _cv2(C.frame(17, 33, "noise"), q)[:R.HEADER_BYTES] == R.header(17, 33, q)


def test_capacity_holds_the_largest_files():
    """q100 noise and saturated frames come closest to the capacity (every block long, many FF bytes)."""
    for h, w in [(16, 16), (97, 131), (480, 854)]:
        for kind in ("noise", "saturated"):
            n = len(_cv2(C.frame(h, w, kind), 100))
            assert n <= R.max_bytes(h, w)
    assert R.max_bytes(480, 854) == 623 + 2 + 2 * -(-9720 * 1660 // 8)


def test_random_shapes_equal_cv2():
    for h, w in C.random_shapes(30):
        f = C.frame(h, w, "smooth", seed=h * w)
        for q in (30, 95):
            assert R.encode(f, q) == _cv2(f, q), (h, w, q)


def test_golden_files_equal_the_restatement():
    g = np.load(GOLDEN)
    for h, w, kind, q in [tuple(int(v) if v.isdigit() else v for v in k.split(":")[1].split("x") + k.split(":")[2:])
                          for k in g.files if k.startswith("jpg:")]:
        want = g[f"jpg:{h}x{w}:{kind}:{q}"].tobytes()
        assert R.encode(C.frame(h, w, kind), q) == want, (h, w, kind, q)


def test_quantisation_reciprocal_is_round_half_away_from_zero():
    """libjpeg-turbo quantises by a reciprocal; over every FDCT output magnitude and every baseline divisor 8 q it
    equals the rounded division the kernel computes."""
    x = np.arange(-(1 << 15), 1 << 15)
    for q in range(1, 256):
        d = 8 * q
        want = np.sign(x) * ((np.abs(x) + d // 2) // d)
        assert np.array_equal(R.quant_divide(x, d), want), q
