"""Whole training runs under --deterministic: the ``train_parent.py --cache device`` run and the streaming
``--loader native`` run give bit-identical checkpoints (the comparison DESIGN.md §15 could only make on printed lines),
and two data-parallel runs at world size 2 give bit-identical parameters."""
import os

import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

from test_gpu_device_frames import _parent_run, tree  # noqa: E402,F401  (fixture and seeded-run helper)


@pytest.fixture
def restore_flag():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield
    torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def test_parent_cache_device_checkpoint_equals_streaming(tree, tmp_path, monkeypatch, capsys, restore_flag):  # noqa: F811
    monkeypatch.setenv("OSVOS_DB_ROOT", tree)
    argv = ["--loader", "native", "--pretrained", "0", "--epochs", "2", "--snapshot", "1", "--test-interval", "1",
            "--n-ave-grad", "1", "--workers", "0", "--val-measures", "--lr", "1e-7", "--deterministic"]
    streamed, fed_s, w_s = _parent_run(argv, tmp_path / "streamed", monkeypatch, capsys)
    cached, fed_c, w_c = _parent_run(argv + ["--cache", "device"], tmp_path / "cached", monkeypatch, capsys)
    assert len(fed_s) == 10 and len(fed_c) == len(fed_s)
    assert len(streamed) == 6 and cached == streamed                   # losses (validation included) and J/F lines
    assert w_s.keys() == w_c.keys()
    for k in w_s:
        assert torch.equal(w_s[k], w_c[k]), k


def _dp_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    import torch.distributed as dist
    from oracle import osvos_oracle as oc
    from osvos_pytorch_b200 import parallel, training
    from osvos_pytorch_b200.networks.vgg_osvos import OSVOS
    torch.use_deterministic_algorithms(True)
    parallel.init_distributed("nccl")
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    net = OSVOS(pretrained=0, verbose=False)
    net.load_state_dict(oc.he_params(seed=0), strict=False)
    net = net.to(dev).train()
    opt = training.make_optimizer(net, "parent", lr=1e-9, fused=True)
    bucket = parallel.GradientBucket(parallel.trainable_parameters(net))
    batches = [training.synthetic_batch(2, 64, 96, 100 * rank + s, dev) for s in range(4)]
    training.parent_epoch(net, opt, bucket, batches, 0, 240, n_ave_grad=2)
    torch.cuda.synchronize()
    torch.save({k: v.cpu() for k, v in net.state_dict().items()}, os.path.join(out, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_dp_world2_runs_are_identical(tmp_path):
    """Same world size, topology and NCCL settings: NCCL's allreduce is reproducible, so the runs are too."""
    world, runs = 2, []
    for r in range(2):
        out = tmp_path / f"run{r}"
        out.mkdir()
        mp.spawn(_dp_worker, args=(world, 29750 + r + os.getpid() % 200, str(out)), nprocs=world, join=True)
        runs.append([torch.load(out / f"rank{k}.pt") for k in range(world)])
    for k in runs[0][0]:
        assert torch.equal(runs[0][0][k], runs[1][0][k]), k
        assert torch.equal(runs[0][0][k], runs[0][1][k]), k                # the replicas stay one model
