"""conv1_1's staged epilogue (registers -> shared memory -> TMA store) against its direct-store epilogue, bit for bit.
TMA stores need 16-byte aligned output planes, so the same launch into planes that start 4 bytes past an aligned address
takes the direct stores with the same arithmetic.  Frames smaller than a tile, odd sizes whose edge tiles the TMA stores
clip, batches, and the 480x854 frame (24 tiles per CTA on a 132-SM H100).
Run on the GPU:  pytest -m gpu."""
import math

import pytest
import torch
import torch.nn.functional as F

from gpu_util import maxrel

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from osvos_pytorch_b200 import _native
    _native.load()
    return torch.device("cuda:0")


@pytest.mark.parametrize("fast", [False, True])
@pytest.mark.parametrize("n,h,w", [(1, 5, 3), (1, 33, 45), (2, 97, 131), (3, 16, 8), (1, 480, 854)])
def test_conv_first_staged_equals_direct_store(dev, n, h, w, fast):
    from osvos_pytorch_b200 import _native as nat, ops
    g = torch.Generator().manual_seed(h * 3 + w)
    x = (torch.rand(n, 3, h, w, generator=g) * 255.0 - 110.0).to(dev)
    w1 = (torch.randn(64, 3, 3, 3, generator=g) * math.sqrt(2.0 / 27)).to(dev)
    b1 = (torch.randn(64, generator=g) * 0.1).to(dev)
    for relu in (True, False):
        y = ops.conv_first(x, w1, b1, relu=relu, fast=fast)
        numel = n * h * w * 64
        bufs = [torch.zeros(numel + 2, dtype=torch.bfloat16, device=dev) for _ in range(2)]
        hi, lo = (t[2:] for t in bufs)                                   # planes at +4 bytes
        flags = (nat.FLAG_RELU if relu else 0) | (nat.FLAG_FAST if fast else 0)
        nat.check(nat.load().osvos_conv_first_fwd(x.data_ptr(), w1.data_ptr(), b1.data_ptr(), hi.data_ptr(),
                                                  None if fast else lo.data_ptr(), n, h, w, flags,
                                                  torch.cuda.current_stream().cuda_stream), "osvos_conv_first_fwd")
        torch.cuda.synchronize()
        assert torch.equal(hi.view(n, h, w, 64), y.hi), relu
        if not fast:
            assert torch.equal(lo.view(n, h, w, 64), y.lo), relu
        ref = F.conv2d(x.double(), w1.double(), b1.double(), padding=1).cpu()
        ref = ref.relu() if relu else ref
        assert maxrel(ops.act_to_nchw(y).cpu(), ref) < (3e-2 if fast else 3e-5), relu
