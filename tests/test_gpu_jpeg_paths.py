"""decode="device" through the data paths that use it: DeviceFrames, SequenceSegmenter(frames="jpeg"),
train_online.py --decode device and train_parent.py --decode device, each against the host-decoding path."""
import gc
import json
import os
import random

import numpy as np
import pytest
import torch

import davis_fixture

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    return davis_fixture.write_tree(davis_fixture.load(), tmp_path_factory.mktemp("davis"))


def _he_net(seed=0):
    import networks.vgg_osvos as vo
    net = vo.OSVOS(pretrained=0, verbose=False)
    vo.he_init_(net, seed=seed)
    with torch.no_grad():
        for mod in list(net.side_prep) + [net.fuse]:
            mod.weight.mul_(0.1)
    return net


@pytest.mark.parametrize("input_res", [None, (40, 56)])
def test_device_frames_with_device_decode_equal_the_host_store(tree, input_res):
    from osvos_pytorch_b200 import davis
    dev = torch.device("cuda")
    for train in (True, False):
        host = davis.DeviceFrames(davis.DAVIS2016Frames(db_root_dir=tree, train=train), dev, input_res=input_res)
        ds = davis.DAVIS2016Frames(db_root_dir=tree, train=train, decode="device")
        store = davis.DeviceFrames(ds, dev, workers=1, input_res=input_res)
        assert store.where == host.where and store.fname == host.fname and store.has_gt == host.has_gt
        for a, b in zip(store.groups, host.groups):
            assert all(torch.equal(a[k], b[k]) for k in ("img", "gt", "stats"))
        assert store.fallback_frames == 0 and store.redecoded_frames == 0


def test_device_frames_redecode_flagged_and_count_fallbacks(tree, tmp_path):
    """A cut-short frame is re-decoded with cv2.imread; a progressive one falls back in the worker."""
    import shutil
    import jpeg_cases
    from osvos_pytorch_b200 import davis
    root = tmp_path / "davis"
    shutil.copytree(tree, root)
    d = davis.DAVIS2016Frames(db_root_dir=str(root), train=True)
    paths = [os.path.join(root, rel) for rel in d.img_list]
    cut = jpeg_cases.cut_short(open(paths[0], "rb").read(), 0.5)
    open(paths[0], "wb").write(cut)
    ok, prog = cv2.imencode(".jpg", cv2.imread(paths[1]), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])
    prog.tofile(paths[1])
    dev = torch.device("cuda")
    host = davis.DeviceFrames(davis.DAVIS2016Frames(db_root_dir=str(root), train=True), dev)
    store = davis.DeviceFrames(davis.DAVIS2016Frames(db_root_dir=str(root), train=True, decode="device"), dev)
    assert store.redecoded_frames == 1 and store.fallback_frames == 1
    for a, b in zip(store.groups, host.groups):
        assert torch.equal(a["img"], b["img"]) and torch.equal(a["gt"], b["gt"])


@pytest.mark.parametrize("opts", [dict(), dict(input_res=(24, 32)), dict(input_res=(24, 32), output_res="stored"),
                                  dict(score=True), dict(score=True, input_res=(24, 32), output_res="stored")])
def test_segmenter_jpeg_equals_bgr8(tree, opts):
    from osvos_pytorch_b200 import davis
    from osvos_pytorch_b200.inference import SequenceSegmenter
    net = _he_net().cuda().eval()
    host = davis.DAVIS2016Frames(db_root_dir=tree, train=False, seq_name="cc", all_annotations=True)
    devd = davis.DAVIS2016Frames(db_root_dir=tree, train=False, seq_name="cc", all_annotations=True, decode="device")
    score = opts.get("score", False)
    hb = [davis.collate([host[i]]) for i in range(len(host))] * 2          # a depth-2 ring comes round twice
    jb = [davis.collate([devd[i]]) for i in range(len(devd))] * 2
    assert all("jpeg" in b for b in jb)

    def bgr8():
        for b in hb:
            img, gt = davis.views(davis.pinned(b["data"]), *(int(v) for v in b["size"]))
            yield (img, gt) if score else img
    a = SequenceSegmenter(net, output="logits", depth=2, frames="bgr8", **opts)
    want = [r.clone() for r in a(bgr8())]
    b = SequenceSegmenter(net, output="logits", depth=2, frames="jpeg", **opts)
    got = [r.clone() for r in b(iter(jb))]
    assert len(got) == len(want) == 2 * len(host)
    assert all(torch.equal(x, y) for x, y in zip(got, want))
    assert int(b.jpeg_status) == 0
    if score:
        assert torch.equal(a.frame_counts(), b.frame_counts())


def test_online_decode_device_writes_the_same_pngs_and_scores(tree, tmp_path, monkeypatch):
    import train_online
    out = {}
    for decode in ("host", "device"):
        save = tmp_path / decode
        save.mkdir()
        torch.save(_he_net(seed=3).state_dict(), save / "parent_epoch-0.pth")
        monkeypatch.setenv("OSVOS_DB_ROOT", tree)
        monkeypatch.setenv("OSVOS_SAVE_ROOT", str(save))
        try:
            train_online.main(["--seq-name", "cc", "--iters", "4", "--n-ave-grad", "2", "--lr", "1e-10", "--seed", "1",
                               "--parent-epoch", "1", "--loader", "native", "--evaluate", "--deterministic",
                               "--decode", decode])
        finally:
            torch.use_deterministic_algorithms(False)
        gc.collect()
        res = save / "Results"
        pngs = {p: open(res / "cc" / p, "rb").read() for p in sorted(os.listdir(res / "cc"))}
        out[decode] = (pngs, json.load(open(res / "cc_scores.json")))
    assert len(out["host"][0]) == 2 and out["device"] == out["host"]


@pytest.mark.parametrize("cache", [[], ["--cache", "device"]])
def test_parent_decode_device_prints_the_same_losses(tree, tmp_path, monkeypatch, capsys, cache):
    import train_parent
    monkeypatch.setenv("OSVOS_DB_ROOT", tree)
    lines = {}
    for decode in ("host", "device"):
        monkeypatch.setenv("OSVOS_SAVE_ROOT", str(tmp_path / decode))
        torch.manual_seed(11)
        random.seed(11)
        try:
            train_parent.main(["--loader", "native", "--pretrained", "0", "--epochs", "2", "--snapshot", "1",
                               "--test-interval", "1", "--n-ave-grad", "1", "--workers", "0", "--val-measures",
                               "--lr", "1e-7", "--deterministic", "--decode", decode] + cache)
        finally:
            torch.use_deterministic_algorithms(False)
        gc.collect()
        out = capsys.readouterr().out.splitlines()
        assert not any(ln.startswith("WARNING") for ln in out)
        lines[decode] = [ln.split("  Execution time")[0] for ln in out if ln.startswith(("[Epoch", "***Testing"))]
    assert len(lines["host"]) == 6 and lines["device"] == lines["host"]
