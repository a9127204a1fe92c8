"""The device JPEG decoder (csrc/jpeg.cu, ops.decode_jpeg) against cv2.imdecode and tests/golden/reference_jpeg.npz,
bit for bit, and the DAVIS data path with decode="device" against the host path and reference_davis.npz."""
import os

import numpy as np
import pytest
import torch

import davis_fixture
import jpeg_cases

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_jpeg.npz")


@pytest.fixture(scope="module")
def files():
    out = dict(jpeg_cases.cv2_matrix())
    out.update(jpeg_cases.pillow_files())
    return out


def _decode(bufs, chunk_bits=0, offset=0):
    from osvos_pytorch_b200 import jpeg, ops
    ps = [jpeg.parse(b) for b in bufs]
    assert all(isinstance(p, jpeg.Parsed) for p in ps)
    blob = jpeg.pack(ps)
    n, h, w = len(ps), ps[0].h, ps[0].w
    dev = torch.from_numpy(blob).cuda()
    store = torch.full((n * h * w * 3 + 16,), 7, dtype=torch.uint8, device="cuda")
    out = store[offset:offset + n * h * w * 3].view(n, h, w, 3)
    _, status = ops.decode_jpeg(dev, n, h, w, out=out, nseg=jpeg.segment_count(blob), chunk_bits=chunk_bits)
    assert int(store[:offset].ne(7).sum()) == 0 and int(store[offset + n * h * w * 3:].ne(7).sum()) == 0
    return out.cpu().numpy(), status.cpu().numpy()


def _cv2(buf):
    return cv2.imdecode(np.frombuffer(buf, np.uint8), cv2.IMREAD_COLOR)


def _by_size(files):
    groups = {}
    for name, buf in files.items():
        groups.setdefault(_cv2(buf).shape[:2], []).append(name)
    return groups


@pytest.mark.parametrize("chunk_bits", [0, 32])
def test_kernel_equals_cv2_over_the_matrix(files, chunk_bits):
    """Every file, batched by size (mixed sampling, tables and restart intervals in one batch)."""
    decoded = set()
    for size, names in _by_size(files).items():
        for b in (1, 3, 12):
            for k0 in range(0, len(names), b):
                batch = names[k0:k0 + b]
                got, status = _decode([files[k] for k in batch], chunk_bits)
                assert (status == 0).all(), (batch, status)
                for i, k in enumerate(batch):
                    assert np.array_equal(got[i], _cv2(files[k])), (k, size, b, chunk_bits)
                    decoded.add((k, b))
    assert decoded == {(k, b) for k in files for b in (1, 3, 12)}


@pytest.mark.parametrize("offset", [1, 2, 3])
def test_unaligned_outputs(files, offset):
    names = ["cv2_420_q75_97x131", "cv2_444_q95_97x131", "cv2_420_rst7"]
    got, status = _decode([files[k] for k in names], 0, offset)
    assert (status == 0).all()
    for i, k in enumerate(names):
        assert np.array_equal(got[i], _cv2(files[k]))


@pytest.mark.parametrize("chunk_bits", [0, 32, 100])
def test_1080p(chunk_bits):
    bufs = [jpeg_cases.cv2_file(jpeg_cases.picture(1080, 1920, seed=s), q, "420") for s, q in ((1, 75), (2, 95))]
    got, status = _decode(bufs, chunk_bits)
    assert (status == 0).all()
    for i, b in enumerate(bufs):
        assert np.array_equal(got[i], _cv2(b))


def test_golden_fixture():
    with np.load(GOLDEN, allow_pickle=False) as z:
        fx = {k: z[k] for k in z.files}
    for key in fx:
        if key.startswith("file:"):
            got, status = _decode([fx[key].tobytes()])
            assert np.array_equal(got[0], fx["bgr:" + key[5:]]), key
            assert (status[0] & 4) == (4 if key == "file:cut_short" else 0), (key, status)
            assert (status[0] & ~4) == 0


@pytest.mark.parametrize("chunk_bits", [0, 32])
def test_cut_short_scan(files, chunk_bits):
    """Scans cut at several points: the kernel equals the restatement everywhere and cv2 where the restatement does
    (a cut inside an MCU's last chroma block is the known exception, DESIGN.md §19), and flags every one."""
    import jpeg_ref
    from osvos_pytorch_b200 import jpeg
    keeps = (0.1, 0.3, 0.45, 0.6, 0.95)
    bufs = [jpeg_cases.cut_short(files["cv2_420_q75_97x131"], keep) for keep in keeps]
    got, status = _decode(bufs, chunk_bits)
    for i, b in enumerate(bufs):
        assert np.array_equal(got[i], jpeg_ref.decode(jpeg.parse(b))[0]), keeps[i]
        if keeps[i] != 0.3:
            assert np.array_equal(got[i], _cv2(b)), keeps[i]
        assert status[i] == 4


def test_inconsistent_header_is_flagged_not_decoded(files):
    from osvos_pytorch_b200 import jpeg, ops
    blob = jpeg.pack([jpeg.parse(files["cv2_420_q75_97x131"])])
    out = torch.zeros((1, 96, 131, 3), dtype=torch.uint8, device="cuda")
    _, status = ops.decode_jpeg(torch.from_numpy(blob).cuda(), 1, 96, 131, out=out, nseg=1)
    assert int(status[0]) == 8 and int(out.sum()) == 0


@pytest.fixture(scope="module")
def fx():
    return davis_fixture.load()


@pytest.fixture(scope="module")
def tree(fx, tmp_path_factory):
    return davis_fixture.write_tree(fx, tmp_path_factory.mktemp("davis"))


def test_to_device_with_device_decode_equals_host_and_reference(fx, tree):
    from osvos_pytorch_b200 import davis
    for mode in (dict(train=True), dict(train=False), dict(train=False, seq_name="aa")):
        host = davis.DAVIS2016Frames(db_root_dir=tree, **mode)
        dev = davis.DAVIS2016Frames(db_root_dir=tree, decode="device", **mode)
        idx = list(range(min(len(host), 3)))
        items = [dev[i] for i in idx]
        assert all("jpeg" in it for it in items)
        status = torch.zeros(1, dtype=torch.int32, device="cuda")
        a = davis.to_device(davis.collate(items), torch.device("cuda"), jpeg_status=status)
        b = davis.to_device(davis.collate([host[i] for i in idx]), torch.device("cuda"))
        assert torch.equal(a["image"], b["image"]) and torch.equal(a["gt"], b["gt"])
        assert int(status) == 0
        img_a, _, _ = davis.upload(davis.collate(items), torch.device("cuda"))
        for k, i in enumerate(idx):
            want_img, _ = davis_fixture.pair(fx, host.img_list[i], items[k]["has_gt"])
            assert np.array_equal(a["image"][k].cpu().numpy().transpose(1, 2, 0), want_img)
            assert np.array_equal(img_a[k].cpu().numpy(), host[i]["image"])


def test_mixed_batch_with_a_progressive_file(tree, tmp_path):
    from osvos_pytorch_b200 import davis
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=True, decode="device")
    items = [d[i] for i in range(3)]
    img = cv2.imread(os.path.join(tree, d.img_list[1]), cv2.IMREAD_COLOR)
    ok, prog = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])
    from osvos_pytorch_b200 import jpeg
    assert isinstance(jpeg.parse(prog.tobytes()), jpeg.Fallback)
    items[1] = {k: v for k, v in items[1].items() if k != "jpeg"}
    items[1]["image"] = cv2.imdecode(prog, cv2.IMREAD_COLOR)
    batch = davis.collate(items)
    assert batch["jpeg"]["device"] == [0, 2] and batch["jpeg"]["fallback"] == [1]
    got, _, _ = davis.upload(batch, torch.device("cuda"), input_res=(240, 427))
    host = davis.DAVIS2016Frames(db_root_dir=tree, train=True)
    want = [host[0]["image"], items[1]["image"], host[2]["image"]]
    ref, _, _ = davis.upload(davis.collate([dict(host[i], image=want[i]) for i in range(3)]), torch.device("cuda"),
                             input_res=(240, 427))
    assert torch.equal(got, ref)
