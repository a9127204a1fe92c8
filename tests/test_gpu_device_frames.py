"""The device-resident frame store on the GPU (davis.DeviceFrames, osvos_affine_warp_u8_indexed): the indexed warp is
the fused warp on the gathered batch bit for bit, the store reproduces the streaming loader's tensors, and
``train_parent.py --cache device`` trains on the same batches as the streaming ``--loader native`` run."""
import gc
import os
import random

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import davis_fixture

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


def _store(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    img = torch.randint(0, 256, (n, h, w, 3), generator=g, dtype=torch.uint8)
    gt = (torch.rand(n, h, w, generator=g) > 0.6).to(torch.uint8) * 255
    for k in range(0, n, 3):                             # every third mask non-binary
        gt[k] = torch.where(torch.rand(h, w, generator=g) > 0.8, 90, gt[k].long()).to(torch.uint8)
    gt[1] = 0                                            # an empty mask
    return img.cuda(), gt.cuda()


@pytest.mark.parametrize("shape", [(9, 33, 45), (40, 24, 31), (5, 97, 131)])
def test_indexed_warp_is_the_warp_of_the_gathered_batch(shape):
    from osvos_pytorch_b200 import augment, ops
    n_store, h, w = shape
    img, gt = _store(n_store, h, w, seed=n_store)
    stats = ops.label_stats_u8(gt)
    binary = set(stats[:, 1].cpu().tolist())
    assert binary == {0, 1}
    rng = random.Random(n_store)
    cases = [list(reversed(range(n_store))),                            # a permutation of the whole store
             [2, 0, 2, 2, n_store - 1, 0],                              # repeats
             [rng.randrange(n_store) for _ in range(33)],               # two launches (32 + 1)
             [n_store - 1]]
    for index in cases:
        params = augment.draw_params(len(index), rng=rng)
        params = [(k % 2 == 0, rot, sc) for k, (_, rot, sc) in enumerate(params)]
        got = augment.affine_warp_u8(img, gt, params, stats, index=index)
        sel = torch.tensor(index, device="cuda")
        want = augment.affine_warp_u8(img[sel].contiguous(), gt[sel].contiguous(), params)
        assert got["image"].shape == (len(index), 3, h, w) and got["gt"].shape == (len(index), 1, h, w)
        assert torch.equal(got["image"], want["image"]), index
        assert torch.equal(got["gt"], want["gt"]), index


def test_indexed_warp_checks_indices_and_stats_on_the_host():
    from osvos_pytorch_b200 import augment, ops
    img, gt = _store(4, 16, 20, seed=1)
    stats = ops.label_stats_u8(gt)
    params = [(False, 0.0, 1.0)]
    for bad in ([4], [-1]):
        with pytest.raises(IndexError):
            augment.affine_warp_u8(img, gt, params, stats, index=bad)
    with pytest.raises(ValueError, match="stats"):
        augment.affine_warp_u8(img, gt, params, index=[0])
    with pytest.raises(ValueError, match="stats"):
        augment.affine_warp_u8(img, gt, params, stats[:3], index=[0])


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    return davis_fixture.write_tree(davis_fixture.load(), tmp_path_factory.mktemp("davis"))


@pytest.mark.parametrize("train,workers,batches", [(True, 0, [[2, 0, 1, 0], [4, 3], [1]]), (False, 2, [[1, 0], [1]])])
def test_store_reproduces_the_streaming_loader(tree, train, workers, batches):
    from osvos_pytorch_b200 import augment, davis
    dev = torch.device("cuda")
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=train)
    store = davis.DeviceFrames(d, dev, workers=workers)
    assert len(store) == len(d)
    items = [d[i] for i in range(len(d))]
    assert store.fname == [it["fname"] for it in items] and store.has_gt == [it["has_gt"] for it in items]
    assert store.nbytes == sum(it["gt"].size * 4 + 8 for it in items)
    rng = random.Random(3)
    for idx in batches:
        params = augment.draw_params(len(idx), rng=rng)
        got = store.augmented(idx, params)
        want = davis.to_device(davis.collate([items[i] for i in idx]), dev, augment=params)
        assert torch.equal(got["image"], want["image"]) and torch.equal(got["gt"], want["gt"]), idx
    for i, it in enumerate(items):
        got = store.ingest(i)
        want = davis.to_device(davis.collate([it]), dev)
        assert torch.equal(got["image"], want["image"]) and torch.equal(got["gt"], want["gt"]), i
        assert torch.equal(got["gt_u8"].cpu(), torch.from_numpy(it["gt"])[None]) and got["fname"] == [it["fname"]]


def test_mixed_size_batch_raises(tree):
    from osvos_pytorch_b200 import davis
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=True)
    store = davis.DeviceFrames(d, torch.device("cuda"))
    assert {g["size"] for g in store.groups} == {(33, 45), (97, 131)}
    with pytest.raises(ValueError, match="share a size"):
        store.augmented([0, 3], [(False, 0.0, 1.0)] * 2)
    with pytest.raises(IndexError):
        store.ingest(len(d))


def test_store_that_does_not_fit_raises_before_allocating(tree, monkeypatch):
    from osvos_pytorch_b200 import davis
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=True)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (1000, 80 * 2 ** 30))
    with pytest.raises(ValueError, match=r"need \d+ bytes .* only 1000 are free"):
        davis.DeviceFrames(d, torch.device("cuda"))
    assert torch.cuda.memory_allocated() == before


def _parent_run(argv, save, monkeypatch, capsys):
    """One seeded train_parent.main run -> (its loss and J/F lines, every batch it trained on, its epoch-1 weights)."""
    import train_parent
    from osvos_pytorch_b200 import training
    fed, parent_epoch = [], training.parent_epoch

    def recording(net, opt, bucket, batches, *args, **kw):
        def batches_seen():
            for b in batches:
                fed.append((b["image"].clone(), b["gt"].clone()))
                yield b
        return parent_epoch(net, opt, bucket, batches_seen(), *args, **kw)
    monkeypatch.setattr(training, "parent_epoch", recording)
    monkeypatch.setenv("OSVOS_SAVE_ROOT", str(save))
    torch.manual_seed(11)
    random.seed(11)
    train_parent.main(argv)
    monkeypatch.setattr(training, "parent_epoch", parent_epoch)
    # the run's network and its engine reference each other, and the engine owns captured CUDA graphs: free them here,
    # not in a garbage collection that happens to run inside a later test's graph capture, which it would invalidate
    gc.collect()
    lines = capsys.readouterr().out.splitlines()
    lines = [ln.split("  Execution time")[0] for ln in lines if ln.startswith(("[Epoch", "***Testing"))]
    return lines, fed, torch.load(save / "parent_epoch-1.pth", map_location="cpu")


def test_parent_cache_device_trains_as_the_streaming_loader(tree, tmp_path, monkeypatch, capsys):
    """Same seeds, same batches: every augmented batch the training step sees is bit-identical to the streaming run's,
    and so are the printed losses and J/F.  The weights agree to the step's own run-to-run variation: its backward
    accumulates with float atomics, so two streaming runs on identical batches already differ in the last bits (about
    1e-4 of a tensor's largest weight after these ten steps)."""
    monkeypatch.setenv("OSVOS_DB_ROOT", tree)
    argv = ["--loader", "native", "--pretrained", "0", "--epochs", "2", "--snapshot", "1", "--test-interval", "1",
            "--n-ave-grad", "1", "--workers", "0", "--val-measures", "--lr", "1e-7"]
    streamed, fed_s, w_s = _parent_run(argv, tmp_path / "streamed", monkeypatch, capsys)
    cached, fed_c, w_c = _parent_run(argv + ["--cache", "device"], tmp_path / "cached", monkeypatch, capsys)
    assert len(fed_s) == 10 and len(fed_c) == len(fed_s)                  # 5 frames x 2 epochs at batch 1
    for k, ((img_s, gt_s), (img_c, gt_c)) in enumerate(zip(fed_s, fed_c)):
        assert torch.equal(img_s, img_c) and torch.equal(gt_s, gt_c), k
    assert len(streamed) == 6 and cached == streamed
    val_losses = [ln for ln in streamed if ln.startswith("***Testing *** Loss")]
    assert len(val_losses) == 2 and val_losses[0] != val_losses[1]          # the weights moved
    # (J and F statistics are NaN here: they skip a sequence's first and last frame, and bb has two)
    assert "nan" not in " ".join(ln for ln in streamed if " Loss " in ln)
    assert w_s.keys() == w_c.keys()
    for k in w_s:
        scale = float(w_s[k].abs().max()) or 1.0
        assert float((w_s[k] - w_c[k]).abs().max()) <= 1e-3 * scale, k


def _dp_worker(rank, world, port, tree, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    from torch.utils.data import DataLoader
    from torch.utils.data.distributed import DistributedSampler
    from osvos_pytorch_b200 import davis, parallel
    parallel.init_distributed("nccl")
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    d = davis.DAVIS2016Frames(db_root_dir=tree, train=True)
    gathered = davis.DeviceFrames(d, dev, group=dist.group.WORLD)
    single = davis.DeviceFrames(d, dev)
    same = gathered.fname == single.fname and gathered.has_gt == single.has_gt
    for i in range(len(d)):
        (g1, s1), (g2, s2) = gathered.where[i], single.where[i]
        a, b = gathered.groups[g1], single.groups[g2]
        same = same and all(torch.equal(a[k][s1], b[k][s2]) for k in ("img", "gt", "stats"))
    sampler = DistributedSampler(d, world, rank, shuffle=True, drop_last=True)
    streaming = DataLoader(d, batch_size=1, sampler=sampler, num_workers=0, drop_last=True, collate_fn=davis.collate)
    index = DataLoader(range(len(d)), batch_size=1, sampler=sampler, num_workers=0, drop_last=True)
    order_equal = True
    for epoch in range(3):
        sampler.set_epoch(epoch)
        want = [b["fname"] for b in streaming]
        got = [[gathered.fname[int(i)] for i in idx] for idx in index]
        order_equal = order_equal and got == want and len(got) == len(d) // world
    torch.save({"same": same, "order": order_equal}, os.path.join(out, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_gathered_store_equals_the_single_process_store(tree, tmp_path):
    world = 2
    mp.spawn(_dp_worker, args=(world, 29700 + os.getpid() % 300, tree, str(tmp_path)), nprocs=world, join=True)
    for r in range(world):
        res = torch.load(tmp_path / f"rank{r}.pt")
        assert res["same"] and res["order"], (r, res)
