"""The JPEG host parser (osvos_pytorch_b200/jpeg.py) and the Python restatement of libjpeg-turbo's decode
(tests/jpeg_ref.py) against cv2.imdecode, bit for bit, and the chunked synchronising Huffman decode the kernel uses
against the sequential one."""
import os

import numpy as np
import pytest

import jpeg_cases
import jpeg_ref
from osvos_pytorch_b200 import jpeg

cv2 = pytest.importorskip("cv2")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_jpeg.npz")


@pytest.fixture(scope="module")
def files():
    out = dict(jpeg_cases.cv2_matrix())
    out.update(jpeg_cases.pillow_files())
    return out


def _check(buf):
    p = jpeg.parse(buf)
    assert isinstance(p, jpeg.Parsed), p
    got, status = jpeg_ref.decode(p)
    want = cv2.imdecode(np.frombuffer(buf, np.uint8), cv2.IMREAD_COLOR)
    return got, status, want


def test_restatement_equals_cv2_on_every_file(files):
    for name, buf in files.items():
        got, status, want = _check(buf)
        assert status == 0, name
        assert np.array_equal(got, want), (name, int((got != want).sum()))


def test_saturated_quality_100_reaches_the_range_limit(files, monkeypatch):
    """The q100 saturated picture drives IDCT outputs outside [0, 255], so the range limit decides those pixels."""
    seen = []
    clip = np.clip

    def spy(a, lo, hi, *args, **kw):
        seen.append(bool(((a < lo) | (a > hi)).any()))
        return clip(a, lo, hi, *args, **kw)
    monkeypatch.setattr(jpeg_ref.np, "clip", spy)
    got, _, want = _check(files["cv2_420_q100_sat"])
    monkeypatch.undo()
    assert seen and seen[0]                            # the first clip call is the luma IDCT's
    assert np.array_equal(got, want)


@pytest.mark.parametrize("keep", [0.1, 0.45, 0.6, 0.8, 0.95])
@pytest.mark.parametrize("name", ["cv2_420_q75_97x131", "cv2_444_q75_97x131", "cv2_420_q75_48x70"])
def test_cut_short_scan_equals_cv2_and_is_flagged(files, name, keep):
    buf = jpeg_cases.cut_short(files[name], keep)
    got, status, want = _check(buf)
    assert np.array_equal(got, want)
    assert status & 4


@pytest.mark.parametrize("name", ["cv2_420_q75_48x70", "cv2_444_q95_33x45", "cv2_422_rst7", "cv2_440_rstrow",
                                  "cv2_gray_48x70", "pil_420_q90"])
@pytest.mark.parametrize("chunk_bits", [32, 77, 512])
def test_chunked_decode_equals_sequential(files, name, chunk_bits):
    p = jpeg.parse(files[name])
    seq, s0 = jpeg_ref.coefficients(p)
    chk, s1 = jpeg_ref.coefficients(p, chunk_bits)
    assert np.array_equal(seq, chk) and s0 == s1 == 0


def test_chunked_decode_of_a_cut_short_scan(files):
    p = jpeg.parse(jpeg_cases.cut_short(files["cv2_420_q75_48x70"], 0.5))
    seq, s0 = jpeg_ref.coefficients(p)
    chk, s1 = jpeg_ref.coefficients(p, 32)
    assert np.array_equal(seq, chk) and s0 == s1 and s0 & 4


@pytest.mark.parametrize("name", list(jpeg_cases.fallback_files()))
def test_parser_reports_fallbacks(name):
    buf, reason = jpeg_cases.fallback_files()[name]
    p = jpeg.parse(buf)
    assert isinstance(p, jpeg.Fallback) and reason in p.reason, p


def test_orientation_1_and_adobe_ycbcr_stay_in_the_subset(files):
    base = files["cv2_420_q75_48x70"]
    for buf in (jpeg_cases.with_app(base, 0xE1, jpeg_cases.exif(1)), jpeg_cases.with_app(base, 0xEE, jpeg_cases.adobe(1))):
        got, _, want = _check(buf)
        assert np.array_equal(got, want)


def test_pack_layout(files):
    ps = [jpeg.parse(files[k]) for k in ("cv2_420_q75_97x131", "cv2_444_q95_97x131", "cv2_420_rst7")]
    blob = jpeg.pack(ps)
    hdr = jpeg.HEADER.unpack_from(blob.tobytes())
    assert hdr[0] == jpeg.MAGIC and hdr[1] == 3 and hdr[2] == sum(len(p.segments) for p in ps)
    assert all(o % 16 == 0 for o in hdr[8:13])
    assert jpeg.segment_count(blob) == hdr[2]
    segs = np.frombuffer(blob[hdr[9]:hdr[9] + hdr[2] * jpeg.SEGMENT.itemsize].tobytes(), jpeg.SEGMENT)
    data = blob[hdr[12]:]
    k = 0
    for p in ps:
        for s in p.segments:
            assert data[segs[k]["byte_off"]:segs[k]["byte_off"] + len(s)].tobytes() == s
            k += 1


def test_golden_fixture_matches_this_cv2_and_the_restatement():
    with np.load(GOLDEN, allow_pickle=False) as z:
        fx = {k: z[k] for k in z.files}
    for key in fx:
        if key.startswith("file:"):
            name = key[5:]
            buf = fx[key].tobytes()
            got, _ = jpeg_ref.decode(jpeg.parse(buf))
            assert np.array_equal(got, fx["bgr:" + name]), name
            assert np.array_equal(cv2.imdecode(fx[key], cv2.IMREAD_COLOR), fx["bgr:" + name]), name
