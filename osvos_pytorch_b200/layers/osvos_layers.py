"""Loss / crop / interpolation helpers with the reference's names and signatures
(layers/osvos_layers.py of kmaninis/OSVOS-PyTorch), the loss running as native
CUDA kernels (csrc/loss.cu) behind a torch.autograd.Function."""
import numpy as np
import torch

from .. import _native as nat


def logit(x):
    """numpy helper, reference layers/osvos_layers.py:11-12."""
    return np.log(x / (1 - x + 1e-08) + 1e-08)


def sigmoid_np(x):
    """numpy helper, reference layers/osvos_layers.py:15-16."""
    return 1 / (1 + np.exp(-x))


def upsample_filt(size):
    """Bilinear tap table of a size x size deconvolution kernel (reference :59-67)."""
    factor = (size + 1) // 2
    center = factor - 1.0 if size % 2 == 1 else factor - 0.5
    taps = 1.0 - np.abs(np.arange(size) - center) / factor
    return taps[:, None] * taps[None, :]


def bilinear_deconv_weight(cin, cout, size):
    """(cin, cout, size, size) tensor with the bilinear table on the diagonal, zeros elsewhere."""
    if cin != cout:
        print('input + output channels need to be the same')
        raise ValueError
    w = torch.zeros(cin, cout, size, size)
    idx = torch.arange(cin)
    w[idx, idx] = torch.from_numpy(upsample_filt(size)).float()
    return w


def interp_surgery(lay):
    """Writes the bilinear taps on the (i, i) diagonal of a ConvTranspose2d weight and returns
    ``lay.weight.data`` (reference :72-85; same ValueError on non-square / mismatched shapes)."""
    m, k, h, w = lay.weight.data.size()
    if m != k:
        print('input + output channels need to be the same')
        raise ValueError
    if h != w:
        print('filters need to be square')
        raise ValueError
    filt = torch.from_numpy(upsample_filt(h)).to(lay.weight.data.dtype)
    with torch.no_grad():
        idx = torch.arange(m)
        lay.weight.data[idx, idx] = filt.to(lay.weight.device)
    return lay.weight.data


def center_crop(x, height, width):
    """Centre crop to (height, width): floor(d/2) removed at the top/left, ceil(d/2) at the
    bottom/right (the negative F.pad of reference :51-56), as a view."""
    dh, dw = x.size(2) - height, x.size(3) - width
    return x[:, :, dh // 2: x.size(2) - (dh - dh // 2), dw // 2: x.size(3) - (dw - dw // 2)]


class _ClassBalancedBCE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, output, label, divisor, void):
        if not output.is_cuda:
            raise RuntimeError("class_balanced_cross_entropy_loss: CUDA tensors required; the H100 package has no "
                               "CPU fallback (oracle/ holds the CPU restatement used by the tests)")
        lib = nat.load()
        x = output.detach().contiguous().float()
        y = label.detach().to(x.device).contiguous().float()
        assert x.numel() == y.numel()
        loss = torch.empty((), dtype=torch.float32, device=x.device)   # 0-dim, not a view: `loss /= k` must work
        stream = torch.cuda.current_stream().cuda_stream
        # deterministic: block sums added in a fixed order instead of with fp64 atomics (rows behind sums[0..4])
        flags = nat.FLAG_DETERMINISTIC if torch.are_deterministic_algorithms_enabled() else 0
        if void:
            flags |= nat.FLAG_VOID_LABELS     # label < 0: void, in neither class (sums[3] = the non-void count)
        sums = torch.empty(lib.osvos_cbce_fwd_sums(x.numel(), flags), dtype=torch.float64, device=x.device)
        nat.check(lib.osvos_cbce_fwd(x.data_ptr(), y.data_ptr(), x.numel(), float(divisor), sums.data_ptr(),
                                     loss.data_ptr(), flags, stream), "osvos_cbce_fwd")
        ctx.save_for_backward(x, y, sums)
        ctx.divisor = float(divisor)
        ctx.void = void
        ctx.shape = output.shape
        return loss

    @staticmethod
    def backward(ctx, grad_out):
        x, y, sums = ctx.saved_tensors
        lib = nat.load()
        g = grad_out.detach().contiguous().float().reshape(1)
        dx = torch.empty_like(x)
        stream = torch.cuda.current_stream().cuda_stream
        bwd = lib.osvos_cbce_bwd_void if ctx.void else lib.osvos_cbce_bwd
        nat.check(bwd(x.data_ptr(), y.data_ptr(), sums.data_ptr(), g.data_ptr(), ctx.divisor, x.numel(), dx.data_ptr(),
                      stream), "osvos_cbce_bwd")
        return dx.reshape(ctx.shape), None, None, None


def class_balanced_cross_entropy_loss(output, label, size_average=True, batch_average=True, void=False):
    """Class-balanced sigmoid BCE (reference :19-48): same arguments, returns a 0-dim tensor that
    supports .item(), /=, .backward(), python sum() and scalar multiplication.

    ``void`` (extension): a label < 0 marks a void pixel (DAVIS-2017's 255), counted in neither class and given zero
    gradient; the class weights then use the non-void count, and an all-void label gives 0.  Not with size_average,
    whose divisor would be that count."""
    if void and size_average:
        raise ValueError("class_balanced_cross_entropy_loss: void=True needs size_average=False")
    if size_average:
        divisor = float(np.prod(label.size()))
    elif batch_average:
        divisor = float(label.size()[0])
    else:
        divisor = 1.0
    return _ClassBalancedBCE.apply(output, label, divisor, bool(void))
