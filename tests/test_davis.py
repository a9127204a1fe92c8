"""CPU checks of the native DAVIS-2016 loader (osvos_pytorch_b200.davis) against the reference dataset's lists
(tests/golden/reference_davis.npz), and of the argument checks of the ingest entry points (csrc/frames.cu)."""
import ctypes

import numpy as np
import pytest
import torch

import davis_fixture

MODES = {"train": dict(train=True), "val": dict(train=False), "seq_train": dict(train=True, seq_name="aa"),
         "seq_test": dict(train=False, seq_name="aa")}


@pytest.fixture(scope="module")
def fx():
    return davis_fixture.load()


@pytest.fixture(scope="module")
def tree(fx, tmp_path_factory):
    return davis_fixture.write_tree(fx, tmp_path_factory.mktemp("davis"))


@pytest.mark.parametrize("mode", sorted(MODES))
def test_file_lists_match_the_reference(fx, tree, mode):
    from osvos_pytorch_b200.davis import DAVIS2016Frames
    d = DAVIS2016Frames(db_root_dir=tree, **MODES[mode])
    assert d.img_list == list(fx[f"list.{mode}.img"])
    assert ["" if v is None else v for v in d.labels] == list(fx[f"list.{mode}.labels"])
    assert len(d) == len(fx[f"list.{mode}.img"])


@pytest.mark.parametrize("mode", ["seq_train", "seq_test"])
def test_sequence_mode_fnames_match_the_reference(fx, tree, mode):
    pytest.importorskip("cv2")
    from osvos_pytorch_b200.davis import DAVIS2016Frames
    d = DAVIS2016Frames(db_root_dir=tree, **MODES[mode])
    assert [d[i]["fname"] for i in range(len(d))] == list(fx[f"list.{mode}.fname"])


def test_items_are_the_reference_decode(fx, tree):
    """The uint8 items, converted on the host the way the reference's make_img_gt_pair does, are its outputs."""
    pytest.importorskip("cv2")
    from osvos_pytorch_b200.davis import DAVIS2016Frames
    mean = np.array((104.00699, 116.66877, 122.67892), dtype=np.float32)
    for mode in ("train", "val", "seq_test"):
        d = DAVIS2016Frames(db_root_dir=tree, **MODES[mode])
        for i in range(len(d)):
            it = d[i]
            assert it["image"].dtype == np.uint8 and it["gt"].dtype == np.uint8
            want_img, want_gt = davis_fixture.pair(fx, d.img_list[i], it["has_gt"])
            assert np.array_equal(np.subtract(np.array(it["image"], np.float32), mean), want_img)
            if it["has_gt"]:
                assert np.array_equal(it["gt"].astype(np.float64) / max(float(it["gt"].max()), 1e-8), want_gt)
            else:
                assert not it["gt"].any() and want_gt.shape == it["gt"].shape


def test_collate_packs_one_buffer(fx, tree):
    pytest.importorskip("cv2")
    from osvos_pytorch_b200 import davis
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=True)
    items = [d[0], d[1]]
    b = davis.collate(items)
    n, h, w = (int(v) for v in b["size"])
    assert (n, h, w) == (2, 33, 45) and b["data"].dtype == torch.uint8 and b["data"].numel() == n * h * w * 4
    img, gt = davis.views(b["data"], n, h, w)
    for i in range(n):
        assert np.array_equal(img[i].numpy(), items[i]["image"]) and np.array_equal(gt[i].numpy(), items[i]["gt"])
    assert b["fname"] == ["aa/00000", "aa/00001"] and b["has_gt"].tolist() == [True, True]
    with pytest.raises(ValueError):
        davis.collate([d[0], d[3]])                          # 33x45 and 97x131


def test_input_res_is_refused(tree):
    from osvos_pytorch_b200.davis import DAVIS2016Frames
    with pytest.raises(NotImplementedError, match="imresize"):
        DAVIS2016Frames(db_root_dir=tree, inputRes=(240, 427))


@pytest.fixture(scope="module")
def lib():
    from osvos_pytorch_b200 import _native as nat
    from osvos_pytorch_b200 import build
    build.build()
    return nat.load()


ADDR = 1 << 20                                           # placeholder device address, never dereferenced


@pytest.mark.parametrize("args,rejected_by", [
    ((None, ADDR, 1, 8, 8), "src != nullptr"),
    ((ADDR, None, 1, 8, 8), "dst != nullptr"),
    ((ADDR, ADDR, 0, 8, 8), "n > 0"),
    ((ADDR, ADDR, 1, 0, 8), "h > 0"),
    ((ADDR, ADDR, 1, 8, 40000), "w < 32768"),
    ((ADDR, ADDR, 70000, 8, 8), "n < 65536"),
])
def test_image_from_bgr8_checks_arguments_first(lib, args, rejected_by):
    assert lib.osvos_image_from_bgr8(*args, 104.0, 116.0, 122.0, None) == 1
    msg = lib.osvos_last_error()
    assert b"invalid argument" in msg and rejected_by.encode() in msg, msg


def test_label_entry_points_check_arguments_first(lib):
    for call, rejected_by in [
        (lambda: lib.osvos_label_stats_u8(None, ADDR, 1, 8, 8, None), "src != nullptr"),
        (lambda: lib.osvos_label_stats_u8(ADDR, None, 1, 8, 8, None), "stats != nullptr"),
        (lambda: lib.osvos_label_stats_u8(ADDR, ADDR, 1, -1, 8, None), "h > 0"),
        (lambda: lib.osvos_label_from_u8(ADDR, None, ADDR, 1, 8, 8, None), "stats != nullptr"),
        (lambda: lib.osvos_label_from_u8(ADDR, ADDR, ADDR, 1, 8, 0, None), "w > 0"),
    ]:
        assert call() == 1
        msg = lib.osvos_last_error()
        assert b"invalid argument" in msg and rejected_by.encode() in msg, msg


def test_affine_warp_u8_checks_arguments_first(lib):
    mats = (ctypes.c_double * 6)(1, 0, 0, 0, 1, 0)
    flips = (ctypes.c_int * 1)(0)
    ok = dict(image_src=ADDR, label_src=ADDR, label_stats=ADDR, image_dst=ADDR, label_dst=ADDR, mats=mats)

    def call(n=1, h=8, w=8, **kw):
        a = dict(ok, **kw)
        return lib.osvos_affine_warp_u8(a["image_src"], a["label_src"], a["label_stats"], a["image_dst"], a["label_dst"],
                                        a["mats"], flips, n, h, w, 104.0, 116.0, 122.0, None)
    for kw, rejected_by in [(dict(mats=None), "inv_matrices_host != nullptr"),
                            (dict(image_src=None, label_src=None, label_stats=None), "image_src != nullptr"),
                            (dict(image_dst=None), "image_dst == nullptr"),
                            (dict(label_stats=None), "label_stats == nullptr"),
                            (dict(label_dst=None), "label_dst == nullptr"),
                            (dict(n=0), "n > 0"), (dict(h=0), "h > 0"), (dict(w=32768), "w < 32768")]:
        assert call(**kw) == 1, kw
        msg = lib.osvos_last_error()
        assert b"invalid argument" in msg and rejected_by.encode() in msg, (kw, msg)
