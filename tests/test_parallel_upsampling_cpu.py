"""The data-parallel plumbing carries the deconvolution weights only when the net learns its upsampling: the gradient
bucket is built from parallel.trainable_parameters, and broadcast_parameters starts every rank from rank 0's
deconvolution weights (world_size 2 over gloo, on a stand-in module as in tests/test_parallel_cpu.py)."""
import os

import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

from osvos_pytorch_b200.parallel import GradientBucket, broadcast_parameters, trainable_parameters


class Tiny(nn.Module):
    def __init__(self, learn):
        super().__init__()
        self.upscale = nn.ModuleList([nn.ConvTranspose2d(1, 1, 4, stride=2, bias=False)])
        self.upscale_ = nn.ModuleList([nn.ConvTranspose2d(1, 1, 4, stride=2, bias=False)])
        self.fuse = nn.Conv2d(4, 1, 1)
        self.learn_upsampling = learn


def _worker(rank, world, port):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        for learn in (False, True):
            torch.manual_seed(rank)                      # different replicas before the broadcast
            net = Tiny(learn)
            names = [n for n, p in net.named_parameters() if any(p is q for q in trainable_parameters(net))]
            assert any(n.startswith("upscale") for n in names) == learn
            bucket = GradientBucket(trainable_parameters(net))
            want = sum(p.numel() for n, p in net.named_parameters() if learn or not n.startswith("upscale"))
            assert bucket.numel == want
            broadcast_parameters(net)
            w = net.upscale[0].weight.detach().clone()
            ref = [torch.empty_like(w) for _ in range(world)]
            dist.all_gather(ref, w)
            assert torch.equal(ref[0], ref[1])
    finally:
        dist.destroy_process_group()


def test_bucket_and_broadcast_with_and_without_learn_upsampling():
    port = 29650 + os.getpid() % 200
    mp.spawn(_worker, args=(2, port), nprocs=2, join=True)
