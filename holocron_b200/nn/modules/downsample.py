"""Pooling modules on the hot path — mirrors holocron/nn/modules/downsample.py (ConcatDownsample2d :26-40, GlobalAvgPool2d :58-77,
GlobalMaxPool2d :80-99, BlurPool2d :106-151, SPP :154-167, ZPool :170-183)."""
from typing import List

import numpy as np
import torch
from torch import Tensor, nn

__all__ = ["BlurPool2d", "ConcatDownsample2d", "GlobalAvgPool2d", "GlobalMaxPool2d", "SPP", "ZPool"]


class ConcatDownsample2d(nn.Module):
    """Stacks adjacent pixels on the channel axis (reference downsample.py:26-40; YOLOv2's pass-through layer)."""

    def __init__(self, scale_factor: int) -> None:
        super().__init__()
        self.scale_factor = scale_factor

    def forward(self, x: Tensor) -> Tensor:
        from ..functional import concat_downsample2d
        return concat_downsample2d(x, self.scale_factor)


class GlobalAvgPool2d(nn.Module):
    """Global average pooling over the spatial dims (RepVGG / ReXNet / Darknet heads, SE blocks).

    bf16 channels_last activations (what the fused conv blocks produce) go through the NHWC pooling kernel with
    fp32 accumulation; any other CUDA tensor goes through the generic row-reduction kernel.
    """

    def __init__(self, flatten: bool = False) -> None:
        super().__init__()
        self.flatten = flatten

    def forward(self, x: Tensor) -> Tensor:
        from .._fused import global_avg_pool_flat
        out = global_avg_pool_flat(x)
        if self.flatten:
            return out
        return out.view(x.size(0), x.size(1), 1, 1)

    def extra_repr(self) -> str:
        return "flatten=True" if self.flatten else ""


class GlobalMaxPool2d(nn.Module):
    """Global max pooling over the spatial dims (reference downsample.py:80-99): (N, C, 1, 1), or (N, C) with
    ``flatten``. bf16 and fp32 inputs run natively (other float dtypes in fp32); the gradient goes to the element
    ``max(dim).indices`` names: the lowest flat index h*W + w among equal maxima, the first NaN of a row holding one."""

    def __init__(self, flatten: bool = False) -> None:
        super().__init__()
        self.flatten = flatten

    def forward(self, x: Tensor) -> Tensor:
        from .._pooling import global_max_pool2d
        out = global_max_pool2d(x)
        return out.view(x.size(0), x.size(1)) if self.flatten else out

    def extra_repr(self) -> str:
        return "flatten=True" if self.flatten else ""


class BlurPool2d(nn.Module):
    """Blur pooling (reference downsample.py:106-151, "Making Convolutional Networks Shift-Invariant Again"): the
    binomial filter of size ``kernel_size`` applied depth-wise with ``stride`` over a reflection padding of
    ((stride - 1) + (kernel_size - 1)) // 2.

    The reflection is folded into the kernel's indices: ``padding`` is kept as the reference's child module but no
    padded copy is made. The taps are the reference's: the outer product of the float64 binomial coefficients, cast to
    the input dtype. Kernel sizes above 7 raise NotImplementedError at forward time (construction and repr match the
    reference for every size); inputs are 4-D."""

    def __init__(self, channels: int, kernel_size: int = 3, stride: int = 2) -> None:
        super().__init__()
        self.channels = channels
        if kernel_size <= 1:
            raise AssertionError
        self.kernel_size = kernel_size
        self.stride = stride
        from .._pooling import blur_padding
        self.padding = nn.ReflectionPad2d([blur_padding(kernel_size, stride)] * 4)  # type: ignore[arg-type]
        self._coeffs = torch.tensor((np.poly1d((0.5, 0.5)) ** (self.kernel_size - 1)).coeffs)

    def forward(self, input_tensor: Tensor) -> Tensor:
        from .._pooling import blur_pool2d
        return blur_pool2d(input_tensor, self._coeffs, self.channels, self.kernel_size, self.stride)

    def extra_repr(self) -> str:
        return f"{self.channels}, kernel_size={self.kernel_size}, stride={self.stride}"


class SPP(nn.ModuleList):
    """Spatial pyramid pooling: cat(x, maxpool_k(x) for k in kernel_sizes) along channels (YOLOv4 neck)."""

    def __init__(self, kernel_sizes: List[int]) -> None:
        super().__init__([nn.MaxPool2d(k_size, stride=1, padding=k_size // 2) for k_size in kernel_sizes])

    def forward(self, x: Tensor) -> Tensor:
        feats = [x] + [pool_layer(x) for pool_layer in self]
        return torch.cat(feats, dim=1)


class ZPool(nn.Module):
    """Z-pooling (reference downsample.py:170-183, "Rotate to Attend: Convolutional Triplet Attention Module"): the max
    and the mean over ``dim``, concatenated along it. 4-D inputs, dim in 1..3 (or its negative form)."""

    def __init__(self, dim: int = 1) -> None:
        super().__init__()
        self.dim = dim

    def forward(self, x: Tensor) -> Tensor:
        from ..functional import z_pool
        return z_pool(x, self.dim)
