"""Data-parallel parent training: one process per GPU, frames sharded across ranks, ONE exchange step
per optimizer step - an allreduce(mean) of the flat fp32 gradient bucket over NCCL (NVLink / NVSwitch).

The reference has no parallelism at all (single gpu_id, train_parent.py:25); its only batch-enlarging
mechanism is gradient accumulation (``loss /= nAveGrad; loss.backward()``, train_parent.py:163-172).
An allreduce-MEAN over R ranks holding one micro-batch each is mathematically the same update as the
reference's nAveGrad = R accumulation (up to fp32 summation order), which is the oracle the DP tests use.
NOTE the class-balance weights of the loss are computed over whatever tensor a rank holds
(layers/osvos_layers.py:30-32), so R ranks x batch b == reference (trainBatch = b, nAveGrad = R),
not reference (trainBatch = R*b).

Design: every trainable gradient lives in ONE contiguous fp32 buffer (``GradientBucket``): ``p.grad`` of
each parameter is a view into it, so autograd accumulates straight into the bucket and the collective
needs no flatten / unflatten copies.  The 349,520 frozen bilinear deconvolution weights (lr = 0 in
both scripts) are excluded: payload = 14,917,637 floats = 59.7 MB per optimizer step.
"""
import os

import torch
import torch.distributed as dist


class GradientBucket:
    def __init__(self, params, device=None):
        self.params = [p for p in params if p.requires_grad]
        device = device or self.params[0].device
        self.numel = sum(p.numel() for p in self.params)
        self.flat = torch.zeros(self.numel, dtype=torch.float32, device=device)
        # measurement aid (bench.py): with time_collective set, every allreduce is bracketed by CUDA events on the current
        # stream; the pairs collect in collective_events (device time of the collective incl. the wait for slower ranks)
        self.time_collective = False
        self.collective_events = []
        self.attach()

    def attach(self):
        """(Re)point every p.grad at its slice of the flat buffer."""
        off = 0
        for p in self.params:
            n = p.numel()
            p.grad = self.flat[off:off + n].view_as(p)
            off += n

    def zero_(self):
        """Replacement for optimizer.zero_grad(): keeps the views alive (set_to_none would drop them)."""
        self.flat.zero_()
        base = self.flat.untyped_storage().data_ptr()
        if any(p.grad is None or p.grad.untyped_storage().data_ptr() != base for p in self.params):
            self.attach()

    def allreduce_mean(self, group=None):
        """The single exchange step of the data-parallel path."""
        if not dist.is_initialized() or dist.get_world_size(group) == 1:
            return None
        world = dist.get_world_size(group)
        ev = None
        if self.time_collective and self.flat.is_cuda:
            ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            ev[0].record()
        if dist.get_backend(group) == "nccl":
            dist.all_reduce(self.flat, op=dist.ReduceOp.AVG, group=group)
        else:                       # gloo (CPU tests) has no AVG
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group)
            self.flat.div_(world)
        if ev is not None:
            ev[1].record()
            self.collective_events.append(ev)
        return self.flat


def trainable_parameters(net):
    """Everything except the deconvolution taps (upscale / upscale_), which are trainable only when the net has
    ``learn_upsampling`` set (backward writes their gradients then)."""
    learn = bool(getattr(net, "learn_upsampling", False))
    return [p for name, p in net.named_parameters() if learn or not name.startswith("upscale")]


def broadcast_parameters(module, src=0, group=None):
    """Make every rank start from rank `src`'s parameters and buffers.  The reference initialises side_prep / score_dsn /
    fuse with an UNSEEDED nn.init.normal_ (networks/vgg_osvos.py:76-83), so independently constructed replicas differ;
    data parallelism is only the reference's nAveGrad accumulation if all replicas are the same model."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    with torch.no_grad():
        for t in list(module.parameters()) + list(module.buffers()):
            dist.broadcast(t.data, src=src, group=group)


def steps_per_rank(total_micro_batches, world, n_ave_grad=1):
    """Micro-batches EVERY rank runs per epoch when `total_micro_batches` are dealt out over `world` ranks: the same on
    all ranks and a multiple of n_ave_grad (as DistributedSampler's drop_last), so that every rank takes part in every
    allreduce - unequal counts would pair gradients of different steps and hang the longer ranks."""
    per = total_micro_batches // world
    return (per // n_ave_grad) * n_ave_grad


def shard_range(total, rank, world):
    """Frames [lo, hi) of a global batch of `total` owned by `rank` (SURVEY.md 8e): contiguous, balanced."""
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def init_distributed(backend=None):
    """torchrun-style rendezvous from RANK / WORLD_SIZE / LOCAL_RANK / MASTER_*; returns (rank, world, local)."""
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29511")
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
            dist.init_process_group(backend, device_id=torch.device("cuda", local))
        else:
            dist.init_process_group(backend)
    return rank, world, local
