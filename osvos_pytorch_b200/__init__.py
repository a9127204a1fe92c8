"""H100-native OSVOS hot path (drop-in for kmaninis/OSVOS-PyTorch's
networks/vgg_osvos.py::OSVOS and layers/osvos_layers.py).

Host code is Python/PyTorch plumbing (parameters, device memory, streams,
autograd glue, torch.distributed); every FLOP of the path runs in the
hand-written sm_90a kernels of csrc/, reached through the C ABI of
include/osvos_b200.h (lib/libosvos_b200.so).  There is no CPU fallback.
"""
from . import _native  # noqa: F401

__all__ = ["_native"]
__version__ = "0.1.0"
