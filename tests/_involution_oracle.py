"""Plain torch restatement of the reference's Involution2d (holocron/nn/modules/conv.py:441-499), differentiable with
autograd and exact in whatever dtype it is given (fp32 against the fixture, fp64 against the kernels). It walks the
K*K taps over a zero-padded input instead of unfolding it. Test and benchmark infrastructure only."""
import torch
import torch.nn.functional as F
from torch import Tensor


def involution2d(x: Tensor, kernel: Tensor, kernel_size: int, stride: int = 1, padding: int = 0, dilation: int = 1,
                 groups: int = 1) -> Tensor:
    """y[n, c, o] = sum_t kernel[n, g(c) * K^2 + t, o] * x[n, c, o * stride - padding + dilation * (i_t, j_t)];
    columns of ``kernel`` past groups * K^2 are ignored."""
    n, c, h, w = x.shape
    k = kernel_size
    ho = (h + 2 * padding - dilation * (k - 1) - 1) // stride + 1
    wo = (w + 2 * padding - dilation * (k - 1) - 1) // stride + 1
    if c % groups != 0 or tuple(kernel.shape[2:]) != (ho, wo):
        raise RuntimeError(f"involution: input {tuple(x.shape)} and kernel {tuple(kernel.shape)} do not match")
    xp = F.pad(x, (padding, padding, padding, padding))
    per_chan = kernel[:, :groups * k * k].reshape(n, groups, 1, k * k, ho, wo)
    per_chan = per_chan.expand(n, groups, c // groups, k * k, ho, wo).reshape(n, c, k * k, ho, wo)
    y = x.new_zeros(n, c, ho, wo)
    for t in range(k * k):
        i, j = divmod(t, k)
        r0, c0 = i * dilation, j * dilation
        window = xp[:, :, r0:r0 + (ho - 1) * stride + 1:stride, c0:c0 + (wo - 1) * stride + 1:stride]
        y = y + per_chan[:, :, t] * window
    return y


def involution_module(x: Tensor, module, dtype=None) -> Tensor:
    """The reference forward of ``module`` (an Involution2d, ours or the reference's) on ``x``, with the parameters cast
    to ``dtype`` (default: x's)."""
    dt = x.dtype if dtype is None else dtype
    s = module.unfold.stride
    kernel = F.avg_pool2d(x, s, s) if s > 1 else x
    kernel = F.conv2d(kernel, module.reduce.weight.to(dt), module.reduce.bias.to(dt))
    kernel = F.conv2d(kernel, module.span.weight.to(dt), module.span.bias.to(dt))
    return involution2d(x, kernel, module.k_size, s, module.unfold.padding, module.unfold.dilation, module.groups)


def involution2d_unfold(x: Tensor, kernel: Tensor, kernel_size: int, stride: int = 1, padding: int = 0,
                        dilation: int = 1, groups: int = 1) -> Tensor:
    """The reference's formulation: the unfolded input (N*C*K^2*Ho*Wo elements) times the broadcast kernel, summed over
    the taps. Used as the eager baseline of tools/involution_bench.py."""
    n, c = x.shape[:2]
    ho, wo = kernel.shape[-2:]
    k2 = kernel_size * kernel_size
    cols = F.unfold(x, kernel_size, dilation, padding, stride).view(n, groups, c // groups, k2, ho, wo)
    return (kernel[:, :groups * k2].reshape(n, groups, 1, k2, ho, wo) * cols).sum(3).reshape(n, c, ho, wo)
