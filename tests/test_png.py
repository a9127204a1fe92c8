"""The numpy restatement of the device PNG encoder (tests/png_ref.py, DESIGN.md §21): its files decode to the input with
Pillow, libpng (cv2) and a plain zlib + unfilter decoder, every CRC and the Adler-32 check out, the row filters are the
heuristic's and the sizes stay close to Pillow's."""
import io
import struct
import zlib

import numpy as np
import pytest

import png_cases as C
import png_ref as P

PIL = pytest.importorskip("PIL.Image")


def _pillow(data):
    return np.array(PIL.open(io.BytesIO(data)))


def _pillow_size(a):
    b = io.BytesIO()
    PIL.fromarray(a, "L").save(b, "PNG")
    return len(b.getvalue())


def _check_file(a, data):
    h, w = a.shape
    cs = P.chunks(data)
    assert [k for k, _, _ in cs] == [b"IHDR"] + [b"IDAT"] * (len(cs) - 2) + [b"IEND"]
    assert all(ok for _, _, ok in cs), "chunk CRC"
    assert cs[0][1] == struct.pack(">IIBBBBB", w, h, 8, 0, 0, 0, 0)
    assert cs[-1][1] == b""
    rows = max(1, P.SEGMENT_BYTES // (w + 1))
    assert len(cs) == 2 + -(-h // rows) + 1                       # one IDAT per segment and the trailer
    assert cs[1][1][:2] == b"\x78\x01"
    trailer = cs[-2][1]
    _, filt = P.filter_rows(a)
    assert trailer[:2] == b"\x03\x00" and struct.unpack(">I", trailer[2:])[0] == zlib.adler32(filt.tobytes())
    assert len(data) <= P.max_bytes(h, w)
    assert np.array_equal(_pillow(data), a)


@pytest.mark.parametrize("shape", C.SHAPES)
@pytest.mark.parametrize("kind", C.KINDS)
def test_files_decode_to_the_input(shape, kind):
    a = C.content(kind, *shape, seed=shape[0] * 7 + shape[1])
    data = P.encode(a)
    _check_file(a, data)
    cv2 = pytest.importorskip("cv2")
    assert np.array_equal(cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_UNCHANGED).reshape(a.shape), a)
    if a.size <= 60000:                                           # the plain decoder unfilters in Python
        got, _ = P.decode(data)
        assert np.array_equal(got, a)


def test_plain_decoder_on_a_full_size_map():
    a = C.bytescale(480, 854, seed=3)
    got, types = P.decode(P.encode(a))
    assert np.array_equal(got, a) and len(set(types.tolist())) >= 2


def _filter_types_by_hand(a):
    """The least-sum-of-residuals choice, written per row and per pixel."""
    a = a.astype(int)
    h, w = a.shape
    out = []
    for y in range(h):
        best = None
        for t in range(5):
            cost = 0
            for x in range(w):
                av = a[y, x - 1] if x else 0
                bv = a[y - 1, x] if y else 0
                cv = a[y - 1, x - 1] if x and y else 0
                p = av + bv - cv
                pa, pb, pc = abs(p - av), abs(p - bv), abs(p - cv)
                pae = av if pa <= pb and pa <= pc else bv if pb <= pc else cv
                pred = (0, av, bv, (av + bv) // 2, pae)[t]
                v = (a[y, x] - pred) & 255
                cost += min(v, 256 - v)
            if best is None or cost < best[0]:
                best = (cost, t)
        out.append(best[1])
    return out


@pytest.mark.parametrize("kind", ["bytescale", "mask", "noise"])
def test_row_filters_are_the_heuristics(kind):
    a = C.content(kind, 23, 41, seed=5)
    _, types = P.decode(P.encode(a))
    assert types.tolist() == _filter_types_by_hand(a)


def test_filters_take_every_type_on_a_mixed_map():
    rng = np.random.default_rng(1)
    a = np.vstack([C.bytescale(40, 60, seed=2), rng.integers(0, 256, (4, 60), dtype=np.uint8),
                   np.tile(np.arange(60, dtype=np.uint8), (4, 1)), C.mask(40, 60, seed=4)])
    _, types = P.decode(P.encode(a))
    assert types.tolist() == _filter_types_by_hand(a)
    assert len(set(types.tolist())) >= 3


def test_runs_are_capped_at_258_with_their_remainders():
    for n in list(range(1, 12)) + [258, 259, 260, 261, 262, 516, 517, 518, 519, 1000]:
        sym, exb, exv, match = P.tokens(np.zeros(n, np.uint8))
        assert int(np.sum(np.where(match == 1, 0, 1))) + sum(                 # every byte accounted for once
            (258 if s == 285 else [r for r in range(3, 259) if P.length_symbol(r)[:1] == (s,)
                                   and P.length_symbol(r)[2] == v][0]) for s, v, m in zip(sym, exv, match) if m) == n
        r = (n - 1) % 258
        assert int(match.sum()) == (0 if n < 4 else (n - 1) // 258 + (r >= 3))
        assert int((match == 0).sum()) == (n if n < 4 else 1 + (r if r < 3 else 0))
        raw = P.segment_data(np.zeros(n, np.uint8), True)[0] + b"\x03\x00" + struct.pack(">I", zlib.adler32(bytes(n)))
        assert zlib.decompress(raw) == bytes(n)


def test_noise_falls_back_to_stored_blocks_within_capacity():
    for h, w in ((240, 427), (480, 854), (5, 8191)):
        a = C.noise(h, w, seed=h)
        data, kinds = P.encode(a, return_blocks=True)
        assert set(kinds) == {"stored"} and len(data) == P.max_bytes(h, w)
        _check_file(a, data)


def test_code_lengths_are_limited_to_15_bits():
    a = C.fibonacci()
    _, filt = P.filter_rows(a)
    sym, _, _, _ = P.tokens(filt.ravel())
    freq = np.bincount(sym, minlength=286).tolist()
    freq[256] = 1
    assert max(P.huffman_lengths(freq, 40)) > 15                  # the unlimited code would be too deep
    limited = P.huffman_lengths(freq, 15)
    assert max(limited) == 15 and sum(2.0 ** -ln for ln in limited if ln) == 1.0   # complete
    data, kinds = P.encode(a, return_blocks=True)
    assert kinds == ["dynamic"]
    _check_file(a, data)
    assert np.array_equal(P.decode(data)[0], a)


def test_code_length_code_is_limited_to_7_bits():
    freq = [0] * 19
    for k, s in enumerate((0, 18, 17, 16, 1, 2, 3, 4, 5, 6)):     # counts 1, 1, 2, 3, 5, ...
        freq[s] = [1, 1, 2, 3, 5, 8, 13, 21, 34, 55][k]
    assert max(P.huffman_lengths(freq, 40)) > 7
    lens = P.huffman_lengths(freq, 7)
    assert max(lens) == 7 and sum(2.0 ** -ln for ln in lens if ln) == 1.0


@pytest.mark.parametrize("shape", [(480, 854), (240, 427)])
@pytest.mark.parametrize("kind", ["bytescale", "mask"])
def test_sizes_within_ten_percent_of_pillow(shape, kind):
    for seed in range(3):
        a = C.content(kind, *shape, seed=seed)
        assert len(P.encode(a)) <= 1.10 * _pillow_size(a)


def test_bytes_are_a_function_of_the_frame():
    a = C.bytescale(97, 131, seed=9)
    assert P.encode(a) == P.encode(a.copy())
    assert P.max_bytes(0, 5) == 0 and P.max_bytes(5, 32768) == 0 and P.max_bytes(32767, 1) > 0
