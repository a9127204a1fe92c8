"""Host side of the device PNG decoder (osvos_pytorch_b200/png.py): parsing, the proposed cuts and their verification
rule (tests/png_inflate_ref.py restates the counting pass), the fallback reasons, packing."""
import struct
import zlib

import numpy as np
import pytest

import png_cases as C
import png_decode_cases as D
import png_inflate_ref as R
import png_ref as P

cv2 = pytest.importorskip("cv2")


def _png():
    from osvos_pytorch_b200 import png
    return png


def _cv(data):
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_GRAYSCALE)


def _unfilter_rows(raw, h, rowbytes):
    """Undo the row filters of `raw` (bpp 1) -> uint8 [h, rowbytes]."""
    rows = np.frombuffer(raw, np.uint8).reshape(h, rowbytes + 1)
    out = np.zeros((h, rowbytes), np.int64)
    for y in range(h):
        t, f = rows[y, 0], rows[y, 1:].astype(np.int64)
        up = out[y - 1] if y else np.zeros(rowbytes, np.int64)
        if t == 0:
            out[y] = f
        elif t == 2:
            out[y] = (f + up) & 255
        else:
            a = c = 0
            for x in range(rowbytes):
                b = up[x]
                if t == 1:
                    pred = a
                elif t == 3:
                    pred = (a + b) >> 1
                else:
                    p = a + b - c
                    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
                    pred = a if pa <= pb and pa <= pc else (b if pb <= pc else c)
                a = out[y, x] = (f[x] + pred) & 255
                c = b
    return out.astype(np.uint8)


@pytest.mark.parametrize("name,data", D.subset_files(), ids=[n for n, _ in D.subset_files()])
def test_parse_geometry_and_stream(name, data):
    png = _png()
    got = png.parse(data)
    assert isinstance(got, png.Parsed), got
    want = _cv(data)
    assert (got.h, got.w) == want.shape
    assert got.depth == (1 if name.startswith(("pillow-1-", "cv2-bilevel")) else 8)
    assert got.stream == D.stream_of(data)
    raw = zlib.decompress(got.stream)
    assert len(raw) == got.h * (got.rowbytes + 1)
    if got.h * got.w <= 6000:                       # the stream is the image: filters undone on the host
        px = _unfilter_rows(raw, got.h, got.rowbytes)
        if got.depth == 1:
            px = np.unpackbits(px, axis=1)[:, :got.w] * 255
        assert np.array_equal(px, want)
    if name.startswith("own-"):
        rows = max(1, P.SEGMENT_BYTES // (got.w + 1))
        assert len(got.cuts) == -(-got.h // rows)       # one per encoder segment; the trailer IDAT follows the last
    else:
        assert all(got.stream[c - 4:c] == D.FLUSH for c in got.cuts)


@pytest.mark.parametrize("shape", D.SMALL + [(240, 427)])
@pytest.mark.parametrize("kind", ["bytescale", "noise"])
def test_own_cuts_are_proven_by_the_counting_rule(shape, kind):
    png = _png()
    got = png.parse(P.encode(C.content(kind, *shape, seed=3)))
    bounds = [2] + got.cuts + [len(got.stream)]
    if shape == (240, 427):                         # zlib only: the plain-Python reader is slow
        parts = [zlib.decompressobj(-15).decompress(got.stream[a:b]) for a, b in zip(bounds, bounds[1:])]
    else:
        parts = []
        for k, (a, b) in enumerate(zip(bounds, bounds[1:])):
            out, clean = R.inflate_segment(got.stream, a, b, last=k == len(bounds) - 2)
            assert clean
            assert out == zlib.decompressobj(-15).decompress(got.stream[a:b])
            parts.append(out)
    assert b"".join(parts) == zlib.decompress(got.stream)


def test_foreign_full_flush_cuts_are_proven():
    png = _png()
    data, m = D.full_flush_file()
    got = png.parse(data)
    assert len(got.cuts) == 3 and np.array_equal(_cv(data), m)
    bounds = [2] + got.cuts + [len(got.stream)]
    parts = [R.inflate_segment(got.stream, a, b, last=k == 3) for k, (a, b) in enumerate(zip(bounds, bounds[1:]))]
    assert all(clean for _, clean in parts)
    assert b"".join(out for out, _ in parts) == zlib.decompress(got.stream)


@pytest.mark.parametrize("make", [D.false_cut_file, D.sync_flush_file])
def test_wrong_hints_are_proposed_and_rejected(make):
    png = _png()
    data, m = make()
    assert np.array_equal(_cv(data), m)
    got = png.parse(data)
    assert len(got.cuts) == 1 and got.stream[got.cuts[0] - 4:got.cuts[0]] == D.FLUSH
    bounds = [2] + got.cuts + [len(got.stream)]
    verdicts = [R.inflate_segment(got.stream, a, b, last=k == 1)[1] for k, (a, b) in enumerate(zip(bounds, bounds[1:]))]
    assert not all(verdicts)


def test_pillow_file_resplit_on_a_chance_flush_pattern():
    """A Pillow file re-split into IDAT chunks so that one ends on 00 00 FF FF inside a block."""
    png = _png()
    m = C.noise(30, 40, 9)
    m[10, 5:9] = [0, 0, 255, 255]
    data = D.pillow(m, compress_level=0)
    stream = D.stream_of(data)
    at = stream.index(D.FLUSH, 8) + 4
    resplit = D.build(30, 40, [stream[:at], stream[at:]])
    assert np.array_equal(_cv(resplit), m)
    got = png.parse(resplit)
    assert got.cuts == [at]
    assert not R.inflate_segment(got.stream, 2, at, last=False)[1]


def test_every_fallback_reason():
    png = _png()
    files = D.fallback_files()
    for reason, data in files.items():
        got = png.parse(data)
        assert isinstance(got, png.Fallback) and got.reason == reason, (reason, got)
    for reason in D.CV2_READS:
        assert _cv(files[reason]) is not None
    assert isinstance(png.parse(b""), png.Fallback)
    assert png.parse(D.build(4, 4, [b"\x78"])).reason == "truncated"
    assert png.parse(D.build(4, 4, [b"\x79\x01" + b"\0" * 8])).reason == "zlib header"
    assert png.parse(D.build(4, 4, [zlib.compress(b"\0" * 12)], depth=4)).reason == "4-bit"


def test_ancillary_chunks_and_any_idat_split():
    png = _png()
    m = C.bytescale(20, 31, 2)
    stream = zlib.compress(D.filtered(m), 6)
    pieces = [stream[:1], stream[1:2], b"", stream[2:9], stream[9:]]
    data = D.build(20, 31, pieces, extra=[(b"gAMA", struct.pack(">I", 45455)), (b"tEXt", b"Comment\0hello")])
    got = png.parse(data)
    assert (got.h, got.w, got.depth, got.stream, got.cuts) == (20, 31, 8, stream, [])
    assert np.array_equal(_cv(data), m)


def test_corrupt_streams_pass_the_parser():
    png = _png()
    files, _ = D.corrupt_files()
    assert all(isinstance(png.parse(f), png.Parsed) for f in files.values())


def test_pack_round_trip():
    png = _png()
    datas = [P.encode(C.bytescale(40, 56, 1)), D.pillow(C.mask(40, 56, 2)), D.pillow(C.mask(40, 56, 3), "1"),
             D.full_flush_file()[0]]
    parsed = [png.parse(d) for d in datas]
    blob = png.pack(parsed)
    assert blob.dtype == np.uint8 and png.segment_count(blob) == sum(len(p.cuts) + 1 for p in parsed)
    magic, n, nseg, h, w, _, _, _, files_off, segs_off, data_off, data_bytes = png.HEADER.unpack_from(blob.tobytes())
    assert (magic, n, h, w) == (png.MAGIC, 4, 40, 56) and files_off % 16 == segs_off % 16 == data_off % 16 == 0
    assert data_off + data_bytes == len(blob)
    files = np.frombuffer(blob, png.FILE, n, files_off)
    segs = np.frombuffer(blob, png.SEGMENT, nseg, segs_off)
    for i, p in enumerate(parsed):
        f = files[i]
        assert (f["h"], f["w"], f["depth"], f["nseg"]) == (40, 56, p.depth, len(p.cuts) + 1)
        lo = data_off + int(f["stream_off"])
        assert blob[lo:lo + int(f["stream_len"])].tobytes() == p.stream
        mine = segs[f["seg0"]:f["seg0"] + f["nseg"]]
        assert list(mine["file"]) == [i] * len(mine) and list(mine["index"]) == list(range(len(mine)))
        assert list(mine["beg"] - f["stream_off"]) == [2] + p.cuts
        assert list(mine["end"] - f["stream_off"]) == p.cuts + [len(p.stream)]
    with pytest.raises(ValueError, match="one size"):
        png.pack(parsed + [png.parse(D.pillow(C.mask(41, 56, 3)))])
    with pytest.raises(ValueError):
        png.pack([])


def test_dataset_scores_is_the_mean_over_sequences():
    import torch
    from osvos_pytorch_b200 import evaluation
    a, b = evaluation.SequenceScores(), evaluation.SequenceScores()
    a.add(torch.tensor([[1, 2, 3, 4, 2, 3]] * 4, dtype=torch.int32))
    b.add(torch.tensor([[1, 1, 2, 2, 2, 2]] * 5, dtype=torch.int32))
    got = evaluation.dataset_scores({"a": a, "b": b})
    ra, rb = a.result()["statistics"], b.result()["statistics"]
    for m in "JF":
        for k in "MOD":
            assert got[m][k] == pytest.approx((ra[m][k] + rb[m][k]) / 2)
    assert got == evaluation.dataset_scores({"a": a.result(), "b": b.result()})
    assert np.isnan(evaluation.dataset_scores({})["J"]["M"])
