"""Lambda layer on the hot path — mirrors holocron/nn/modules/lambda_layer.py:15-108. Parameter names / shapes, children
and construction order are the reference's (state_dict and seeded-init contract)."""
from typing import Optional

import torch
from torch import Tensor, nn

__all__ = ["LambdaLayer"]


class LambdaLayer(nn.Module):
    """Lambda layer (LambdaNetworks, https://openreview.net/pdf?id=xTJEN-ggl1b): queries attend to a per-sample linear
    function of the context instead of to every position. ``q = norm_q(to_q(x))``, ``v = norm_v(to_v(x))``, the keys
    ``to_k(x)`` are softmax-normalised over the positions; the content lambda is ``sum_m softmax(k) v``, the position lambda
    a correlation of v with ``R`` (local contexts of odd size ``r``) or a product with ``pos_emb`` (global, ``n`` = H*W
    positions), and the output ``q`` contracted with both.

    Children ``to_q, to_k, to_v, norm_q, norm_v`` and the parameter ``R`` / ``pos_emb`` as in the reference, created in its
    order (same seeded init and ``state_dict``). The three 1x1 projections run on the tensor-core convolution and the two
    BatchNorms on the fused BatchNorm pass; the lambdas and the output run on kernels of their own
    (:mod:`holocron_b200.nn._lambda`), which never build the B x dim_k x dim_v x H x W position lambda of the local
    variant. A bf16 channels_last input takes no layout copy; other dtypes run in bf16 and the output is cast back.
    A global layer fed an input whose H*W differs from ``n`` raises RuntimeError before any launch, as the reference
    fails there; dim_k outside {8, 16, 32}, dim_u > 4, more than 8 heads or r > 23 raise NotImplementedError.
    """

    def __init__(self, in_channels: int, out_channels: int, dim_k: int, n: Optional[int] = None, r: Optional[int] = None,
                 num_heads: int = 4, dim_u: int = 1) -> None:
        super().__init__()
        self.u = dim_u
        self.num_heads = num_heads
        if out_channels % num_heads != 0:
            raise AssertionError("values dimension must be divisible by number of heads for multi-head query")
        dim_v = out_channels // num_heads
        self.to_q = nn.Conv2d(in_channels, dim_k * num_heads, 1, bias=False)
        self.to_k = nn.Conv2d(in_channels, dim_k * dim_u, 1, bias=False)
        self.to_v = nn.Conv2d(in_channels, dim_v * dim_u, 1, bias=False)
        self.norm_q = nn.BatchNorm2d(dim_k * num_heads)
        self.norm_v = nn.BatchNorm2d(dim_v * dim_u)
        self.local_contexts = r is not None
        if r is not None:
            if r % 2 != 1:
                raise AssertionError("Receptive kernel size should be odd")
            self.padding = r // 2
            self.R = nn.Parameter(torch.randn(dim_k, dim_u, 1, r, r))
        else:
            if n is None:
                raise AssertionError("You must specify the total sequence length (h x w)")
            self.pos_emb = nn.Parameter(torch.randn(n, n, dim_k, dim_u))

    def forward(self, x: Tensor) -> Tensor:
        from .. import _fused as K
        from .._lambda import check_lambda, lambda_layer
        _, _, h, w = x.shape
        dim_k = self.to_k.out_channels // self.u
        dim_v = self.to_v.out_channels // self.u
        r = self.R.shape[-1] if self.local_contexts else None
        if not self.local_contexts and h * w != self.pos_emb.shape[1]:
            raise RuntimeError(f"LambdaLayer: a {h}x{w} input has {h * w} positions, pos_emb was built for "
                               f"{self.pos_emb.shape[1]}")
        check_lambda(dim_k, self.u, self.num_heads, r)
        xb = K.to_channels_last_bf16(x, K.round_up(x.shape[1], 8))   # the projections read 8-channel vectors
        q = K.bn_act([K.conv2d(xb, self.to_q.weight, keep_padded=True)], [self.norm_q])
        k = K.conv2d(xb, self.to_k.weight, keep_padded=True)
        v = K.bn_act([K.conv2d(xb, self.to_v.weight, keep_padded=True)], [self.norm_v])
        y = lambda_layer(q, k, v, self.R if self.local_contexts else self.pos_emb, dim_k, self.u, self.num_heads, dim_v, r)
        return y if x.dtype == torch.bfloat16 else y.to(x.dtype)
