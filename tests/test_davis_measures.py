"""CPU checks of the DAVIS-2016 J and F scoring: known answers of the numpy oracle (tests/davis_measures_ref.py),
osvos_pytorch_b200.evaluation against it, the argument checks of osvos_davis_measures, the all-annotations sequence
lists and the refusals of ``train_online.py --evaluate``."""
import math

import numpy as np
import pytest
import torch

import davis_fixture
import davis_measures_ref as ref


def square(h, w, y0, x0, s):
    m = np.zeros((h, w), dtype=bool)
    m[y0:y0 + s, x0:x0 + s] = True
    return m


def jf(p, g, r=None):
    return ref.j_and_f(ref.counts(np.where(p, 1.0, -1.0).astype(np.float32), g.astype(np.uint8) * 255, r))


def test_identical_and_empty_masks():
    m = square(40, 50, 10, 12, 9)
    assert jf(m, m) == (1.0, 1.0)
    empty = np.zeros((40, 50), dtype=bool)
    assert jf(empty, empty) == (1.0, 1.0)
    assert jf(empty, m) == (0.0, 0.0)
    full = np.ones((40, 50), dtype=bool)
    assert ref.seg2bmap(full).sum() == 0
    assert jf(full, full) == (1.0, 1.0)


@pytest.mark.parametrize("s", [1, 2, 5, 16])
def test_square_has_4s_boundary_pixels(s):
    assert ref.seg2bmap(square(40, 50, 10, 12, s)).sum() == 4 * s


@pytest.mark.parametrize("shift", [1, 3, 4, 5, 8])
def test_shifted_square(shift):
    h, w, s = 60, 80, 20
    r = 4
    g = square(h, w, 20, 20, s)
    p = square(h, w, 20, 20 + shift, s)
    j, f = jf(p, g, r)
    assert j == (s - shift) * s / ((s + shift) * s)
    if shift <= r:
        assert f == 1.0
    else:
        assert f < 1.0


def test_disk_and_bound_pix():
    d = ref.disk(8)
    assert d.sum() == 197
    assert [int(d[i].sum() - 1) // 2 for i in range(9)] == [0, 3, 5, 6, 6, 7, 7, 7, 8]
    from osvos_pytorch_b200.evaluation import bound_pix
    for (h, w), r in {(480, 854): 8, (1080, 1920): 18, (240, 427): 4, (720, 1280): 12}.items():
        assert bound_pix(h, w) == ref.bound_pix(h, w) == r


def test_statistics():
    from osvos_pytorch_b200 import evaluation
    assert evaluation.decay_bins(10).tolist() == [0, 2, 5, 7, 9]
    inner = [0.9, 0.8, 0.7, 0.6, 0.55, 0.5, 0.45, 0.4, 0.2, 0.1]
    series = [1.0] + inner + [0.0]                       # the first and last frame are left out
    st = evaluation.statistics(series)
    assert st["M"] == pytest.approx(np.mean(inner))
    assert st["O"] == pytest.approx(5 / 10)
    assert st["D"] == pytest.approx(np.mean(inner[0:3]) - np.mean(inner[7:10]))
    assert (st["M"], st["O"], st["D"]) == ref.statistics(series)
    for short in ([], [0.3], [0.3, 0.4]):
        assert all(math.isnan(v) for v in evaluation.statistics(short).values())
        assert all(math.isnan(v) for v in ref.statistics(short))
    assert evaluation.statistics(torch.tensor([0.0, 0.7, 0.0], dtype=torch.float64)) == {"M": 0.7, "O": 1.0, "D": 0.0}


def test_j_and_f_match_the_oracle():
    from osvos_pytorch_b200 import evaluation
    rng = np.random.default_rng(0)
    rows = [[0, 0, 0, 0, 0, 0], [0, 10, 0, 12, 0, 0], [10, 10, 12, 0, 0, 0], [5, 12, 8, 8, 8, 8], [0, 30, 9, 7, 0, 0]]
    for _ in range(50):
        n_fg, n_gt = rng.integers(0, 40, 2)
        union = int(rng.integers(0, 500))
        rows.append([int(rng.integers(0, union + 1)), union, int(n_fg), int(n_gt), int(rng.integers(0, n_fg + 1)),
                     int(rng.integers(0, n_gt + 1))])
    c = torch.tensor(rows, dtype=torch.int32)
    j, f = evaluation.j_and_f(c)
    want = np.array([ref.j_and_f(r) for r in rows])
    assert np.array_equal(j.numpy(), want[:, 0]) and np.array_equal(f.numpy(), want[:, 1])

    acc = evaluation.SequenceScores()
    for k in range(0, len(rows), 7):
        acc.add(c[k:k + 7])
    res = acc.result()
    assert res["counts"] == rows and res["J"] == want[:, 0].tolist() and res["F"] == want[:, 1].tolist()
    assert tuple(res["statistics"]["F"].values()) == ref.statistics(want[:, 1])


@pytest.fixture(scope="module")
def lib():
    from osvos_pytorch_b200 import _native as nat
    from osvos_pytorch_b200 import build
    build.build()
    return nat.load()


ADDR = 1 << 20                                           # placeholder device address, never dereferenced


@pytest.mark.parametrize("args,rejected_by", [
    ((None, ADDR, ADDR, ADDR, 1, 8, 8, 1), "logits != nullptr"),
    ((ADDR, None, ADDR, ADDR, 1, 8, 8, 1), "masks != nullptr"),
    ((ADDR, ADDR, None, ADDR, 1, 8, 8, 1), "counts != nullptr"),
    ((ADDR, ADDR, ADDR, None, 1, 8, 8, 1), "workspace != nullptr"),
    ((ADDR, ADDR, ADDR, ADDR, 0, 8, 8, 1), "n > 0"),
    ((ADDR, ADDR, ADDR, ADDR, 1, -1, 8, 1), "h > 0"),
    ((ADDR, ADDR, ADDR, ADDR, 1, 8, 0, 1), "w > 0"),
    ((ADDR, ADDR, ADDR, ADDR, 1, 8, 8, 0), "r >= 1"),
    ((ADDR, ADDR, ADDR, ADDR, 1, 8, 8, 32), "r <= OSVOS_DAVIS_MAX_RADIUS"),
    ((ADDR + 2, ADDR, ADDR, ADDR, 1, 8, 8, 1), "& 3) == 0"),
])
def test_davis_measures_checks_arguments_first(lib, args, rejected_by):
    assert lib.osvos_davis_measures(*args, None) == 1
    msg = lib.osvos_last_error()
    assert b"invalid argument" in msg and rejected_by.encode() in msg, msg


def test_workspace_query(lib):
    from osvos_pytorch_b200 import _native as nat
    assert lib.osvos_davis_measures_workspace_bytes(12, 480, 854) == 4 * 4 * 12 * 480 * 27
    assert lib.osvos_davis_measures_workspace_bytes(0, 480, 854) == 0
    assert nat.DAVIS_MAX_RADIUS >= 18


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    return davis_fixture.write_tree(davis_fixture.load(), tmp_path_factory.mktemp("davis"))


def test_all_annotations_lists_every_mask(tree):
    pytest.importorskip("cv2")
    import os
    from osvos_pytorch_b200.davis import DAVIS2016Frames
    d = DAVIS2016Frames(db_root_dir=tree, train=False, seq_name="aa", all_annotations=True)
    assert d.labels == [f"Annotations/480p/aa/{i:05d}.png" for i in range(3)]
    items = [d[i] for i in range(len(d))]
    assert all(it["has_gt"] for it in items) and [it["fname"] for it in items] == ["aa/00000", "aa/00001", "aa/00002"]
    default = DAVIS2016Frames(db_root_dir=tree, train=False, seq_name="aa")
    assert default.labels[1:] == [None, None] and d.img_list == default.img_list
    assert np.array_equal(items[0]["gt"], default[0]["gt"]) and items[2]["gt"].any()
    os.remove(os.path.join(tree, "Annotations/480p/bb/00001.png"))
    try:
        with pytest.raises(ValueError, match="2 frames but 1 annotations"):
            DAVIS2016Frames(db_root_dir=tree, train=False, seq_name="bb", all_annotations=True)
    finally:
        davis_fixture.write_tree(davis_fixture.load(), tree)


@pytest.mark.parametrize("extra,message", [(["--synthetic"], "--synthetic"), ([], "--loader reference"),
                                           (["--loader", "reference"], "--loader reference")])
def test_online_evaluate_needs_the_native_loader(extra, message, capsys):
    import train_online
    with pytest.raises(SystemExit):
        train_online.main(["--evaluate"] + extra)
    assert message in capsys.readouterr().err


def test_parent_val_measures_needs_the_native_loader(capsys):
    import train_parent
    with pytest.raises(SystemExit):
        train_parent.parse(["--val-measures", "--synthetic"])
    assert "--synthetic" in capsys.readouterr().err
    assert train_parent.parse(["--val-measures", "--loader", "native"]).val_measures
