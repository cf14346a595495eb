"""Attention layers (reference holocron/nn/modules/attention.py): the module trees, parameter names and construction
order of the reference, so its checkpoints load unchanged and seeded initialisations match. The forward methods do not
run the children: they hand the children's parameters and buffers to the fused CUDA functions of ``nn/_attention.py``."""
import torch.nn as nn
from torch import Tensor

from .downsample import ZPool

__all__ = ["SAM", "TripletAttention"]


class SAM(nn.Module):
    """SAM layer from `"CBAM: Convolutional Block Attention Module" <https://arxiv.org/pdf/1807.06521.pdf>`_ modified
    in `"YOLOv4: Optimal Speed and Accuracy of Object Detection" <https://arxiv.org/pdf/2004.10934.pdf>`_: x gated by
    sigmoid(conv1x1(x)) per pixel.

    Args:
        in_channels (int): input channels
    """

    def __init__(self, in_channels: int) -> None:
        super().__init__()
        self.conv = nn.Conv2d(in_channels, 1, 1)

    def forward(self, x: Tensor) -> Tensor:
        from .._attention import sam
        return sam(x, self.conv.weight, self.conv.bias)


class DimAttention(nn.Module):
    """Attention layer across a specific dimension: x gated by sigmoid(BN(conv7x7(z_pool(x)))), z_pool taken over
    ``dim`` (1..3, or its negative form).

    Args:
        dim: dimension to compute attention on
    """

    def __init__(self, dim: int) -> None:
        super().__init__()
        self.compress = nn.Sequential(
            ZPool(dim=1),
            nn.Conv2d(2, 1, kernel_size=7, stride=1, padding=3, bias=False),
            nn.BatchNorm2d(1, eps=1e-5, momentum=0.01),
            nn.Sigmoid(),
        )
        self.dim = dim

    def branch(self):
        """(dim, convolution, BatchNorm2d) of this branch, as the fused function takes it."""
        return self.dim, self.compress[1], self.compress[2]

    def forward(self, x: Tensor) -> Tensor:
        from .._attention import triplet_attention
        return triplet_attention(x, [self.branch()])


class TripletAttention(nn.Module):
    """Triplet attention layer from `"Rotate to Attend: Convolutional Triplet Attention Module"
    <https://arxiv.org/pdf/2010.03045.pdf>`_: the mean of the C, H and W branches, all three computed by the same
    launches.
    """

    def __init__(self) -> None:
        super().__init__()
        self.c_branch = DimAttention(dim=1)
        self.h_branch = DimAttention(dim=2)
        self.w_branch = DimAttention(dim=3)

    def forward(self, x: Tensor) -> Tensor:
        from .._attention import triplet_attention
        return triplet_attention(x, [self.c_branch.branch(), self.h_branch.branch(), self.w_branch.branch()])
