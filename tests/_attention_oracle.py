"""Plain-torch restatement of the reference's attention layers (holocron/nn/modules/attention.py): SAM, DimAttention
and TripletAttention, with the transposes, z_pool, convolution, BatchNorm and sigmoid as separate torch ops. It runs in
whatever dtype it is given (fp64 for the GPU parity tests) and on any device; tests/golden/attention.pt pins it to the
unmodified reference."""
from typing import Dict, Optional

import torch
import torch.nn.functional as F
from torch import Tensor


def z_pool(x: Tensor, dim: int) -> Tensor:
    return torch.cat([x.max(dim, keepdim=True).values, x.mean(dim, keepdim=True)], dim=dim)


def sam(x: Tensor, weight: Tensor, bias: Tensor) -> Tensor:
    return x * torch.sigmoid(F.conv2d(x, weight, bias))


def dim_attention(x: Tensor, dim: int, p: Dict[str, Tensor], training: bool, momentum: float = 0.01,
                  eps: float = 1e-5) -> Tensor:
    """One branch. ``p``: conv_weight, bn_weight, bn_bias, running_mean, running_var (the running statistics are
    updated in place in training, like the module's buffers)."""
    if dim != 1:
        x = x.transpose(dim, 1).contiguous()
    z = F.conv2d(z_pool(x, 1), p["conv_weight"], padding=3)
    g = torch.sigmoid(F.batch_norm(z, p["running_mean"], p["running_var"], p["bn_weight"], p["bn_bias"], training,
                                   momentum, eps))
    out = x * g
    if dim != 1:
        out = out.transpose(dim, 1).contiguous()
    return out


def triplet_attention(x: Tensor, branches: Dict[str, Dict[str, Tensor]], training: bool) -> Tensor:
    """``branches``: {"c": params, "h": params, "w": params} as dim_attention takes them."""
    x_c = dim_attention(x, 1, branches["c"], training)
    x_h = dim_attention(x, 2, branches["h"], training)
    x_w = dim_attention(x, 3, branches["w"], training)
    return (x_c + x_h + x_w) / 3


def branch_params(mod, dtype: Optional[torch.dtype] = None, device=None) -> Dict[str, Tensor]:
    """Copies of a DimAttention's parameters and running statistics (leaf tensors requiring grad for the parameters)."""
    conv, bn = mod.compress[1], mod.compress[2]

    def cp(t, grad):
        t = t.detach().clone().to(dtype=dtype or t.dtype, device=device or t.device)
        return t.requires_grad_(grad)

    return {"conv_weight": cp(conv.weight, True), "bn_weight": cp(bn.weight, True), "bn_bias": cp(bn.bias, True),
            "running_mean": cp(bn.running_mean, False), "running_var": cp(bn.running_var, False)}
