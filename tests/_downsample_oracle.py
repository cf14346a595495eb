"""Plain torch restatement of the reference's BlurPool2d, GlobalMaxPool2d and z_pool (holocron/nn/modules/downsample.py
:80-151, holocron/nn/functional.py:139-147), forward and backward written out, in whatever dtype it is given (fp32 / bf16
against the fixture, fp64 against the kernels). The blur walks the K*K taps over reflected indices instead of padding
the input; the max states its index rule explicitly. Test and benchmark infrastructure only."""
from typing import Tuple

import numpy as np
import torch
from torch import Tensor


def blur_filter(kernel_size: int, dtype: torch.dtype) -> Tensor:
    """The reference's 2-D filter: the outer product of the float64 binomial coefficients, cast to ``dtype``."""
    c = torch.tensor((np.poly1d((0.5, 0.5)) ** (kernel_size - 1)).coeffs)
    return (c[:, None] * c[None, :]).to(dtype)


def _reflect(t: Tensor, n: int) -> Tensor:
    return torch.where(t < 0, -t, torch.where(t >= n, 2 * (n - 1) - t, t))


def _taps(h: int, w: int, k: int, s: int, device):
    """For each tap (i, j): the reflected source rows [Ho] and columns [Wo] of the output grid."""
    p = ((s - 1) + (k - 1)) // 2
    ho, wo = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    oy, ox = torch.arange(ho, device=device) * s - p, torch.arange(wo, device=device) * s - p
    return [(i, j, _reflect(oy + i, h), _reflect(ox + j, w)) for i in range(k) for j in range(k)], (ho, wo)


def blur_pool2d(x: Tensor, k: int, s: int, filt: Tensor = None) -> Tensor:
    """y[n, c, oy, ox] = sum_{i,j} f[i, j] * x[n, c, r(oy*s - p + i), r(ox*s - p + j)], accumulated in x's dtype (fp64 in,
    fp64 sums) or in fp32 for narrower inputs, then cast to x's dtype."""
    acc_t = torch.float64 if x.dtype == torch.float64 else torch.float32
    f = blur_filter(k, x.dtype) if filt is None else filt
    taps, (ho, wo) = _taps(x.shape[2], x.shape[3], k, s, x.device)
    xa = x.to(acc_t)
    y = xa.new_zeros(x.shape[0], x.shape[1], ho, wo)
    for i, j, rows, cols in taps:
        y = y + f[i, j].item() * xa[:, :, rows][:, :, :, cols]
    return y.to(x.dtype)


def blur_pool2d_backward(dy: Tensor, in_shape: Tuple[int, ...], k: int, s: int, filt: Tensor = None) -> Tensor:
    """The adjoint of blur_pool2d: every tap scatters f[i, j] * dy onto its reflected source pixel."""
    acc_t = torch.float64 if dy.dtype == torch.float64 else torch.float32
    f = blur_filter(k, dy.dtype) if filt is None else filt
    n, c, h, w = in_shape
    taps, _ = _taps(h, w, k, s, dy.device)
    dx = torch.zeros(n, c, h * w, dtype=acc_t, device=dy.device)
    d = dy.to(acc_t)
    for i, j, rows, cols in taps:
        flat = (rows[:, None] * w + cols[None, :]).flatten()
        dx.index_add_(2, flat, (f[i, j].item() * d).reshape(n, c, -1))
    return dx.view(n, c, h, w).to(dy.dtype)


def max_index(x: Tensor, dim: int) -> Tensor:
    """The index max(dim).indices names: the first NaN of a row holding one, otherwise the first maximum."""
    nan = torch.isnan(x)
    has_nan = nan.any(dim, keepdim=True)
    amax = torch.where(nan, torch.full_like(x, float("-inf")), x).amax(dim, keepdim=True)
    hit = torch.where(has_nan, nan, x == amax)
    return hit.to(torch.int8).argmax(dim, keepdim=True)


def z_pool(x: Tensor, dim: int) -> Tuple[Tensor, Tensor]:
    """(cat([max, mean], dim), the max's index); the mean is summed in fp64 and cast to x's dtype."""
    idx = max_index(x, dim)
    mx = x.gather(dim, idx)
    mean = x.double().sum(dim, keepdim=True).div(x.shape[dim]).to(x.dtype)
    return torch.cat([mx, mean], dim), idx


def z_pool_backward(dy: Tensor, idx: Tensor, x_shape: Tuple[int, ...], dim: int) -> Tensor:
    """dx = dmax at the max's index + dmean / L, each term in dy's dtype as autograd forms it."""
    dmax, dmean = dy.split(1, dim)
    dx = (dmean / x_shape[dim]).expand(x_shape).clone()
    return dx.scatter_add(dim, idx, dmax)


def global_max_pool2d(x: Tensor) -> Tuple[Tensor, Tensor]:
    """((N, C, 1, 1) max over H*W, its flat index h*W + w)."""
    flat = x.reshape(x.shape[0], x.shape[1], -1)
    idx = max_index(flat, 2)
    return flat.gather(2, idx).unsqueeze(-1), idx


def global_max_pool2d_backward(dy: Tensor, idx: Tensor, x_shape: Tuple[int, ...]) -> Tensor:
    n, c, h, w = x_shape
    dx = torch.zeros(n, c, h * w, dtype=dy.dtype, device=dy.device)
    return dx.scatter(2, idx, dy.reshape(n, c, 1)).view(n, c, h, w)
