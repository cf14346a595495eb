"""Plain torch restatement of the reference's LambdaLayer (holocron/nn/modules/lambda_layer.py:15-108), differentiable with
autograd and exact in whatever dtype it is given (fp32 against the fixture, fp64 against the kernels). The local position
term walks the r*r taps over the zero-padded values with the per-tap query product Qr = sum_k q R. Test and benchmark
infrastructure only."""
from typing import Optional

import torch
import torch.nn.functional as F
from torch import Tensor


def lambda_core(q: Tensor, k: Tensor, v: Tensor, pos: Tensor, dim_k: int, dim_u: int, num_heads: int,
                r: Optional[int]) -> Tensor:
    """q [B, heads*dk, H, W] (channel h*dk+k), k [B, dk*u, H, W] (k*u+u'), v [B, dv*u, H, W] (v*u+u'); ``pos`` is R
    [dk, u, 1, r, r] when ``r`` is given, pos_emb [n, n, dk, u] otherwise. Returns y [B, heads*dv, H, W] (h*dv+v)."""
    b, _, h, w = q.shape
    n = h * w
    u = dim_u
    dv = v.shape[1] // u
    qh = q.reshape(b, num_heads, dim_k, n)
    sig = k.reshape(b, dim_k, u, n).softmax(-1)
    vv = v.reshape(b, dv, u, n)
    lc = torch.einsum("bkum,bvum->bkv", sig, vv)
    y = torch.einsum("bhkn,bkv->bhvn", qh, lc)
    if r is not None:
        p = r // 2
        vp = F.pad(v.reshape(b, dv * u, h, w), (p, p, p, p)).reshape(b, dv, u, h + 2 * p, w + 2 * p)
        rw = pos.reshape(dim_k, u, r, r)
        for i in range(r):
            for j in range(r):
                qr = torch.einsum("bhkn,ku->bhun", qh, rw[:, :, i, j])
                win = vp[..., i:i + h, j:j + w].reshape(b, dv, u, n)
                y = y + torch.einsum("bhun,bvun->bhvn", qr, win)
    else:
        if pos.shape[1] != n:
            raise RuntimeError(f"lambda: {n} positions, pos_emb built for {pos.shape[1]}")
        lp = torch.einsum("nmku,bvum->bnkv", pos, vv)
        y = y + torch.einsum("bhkn,bnkv->bhvn", qh, lp)
    return y.reshape(b, num_heads * dv, h, w)


def lambda_core_conv3d(q: Tensor, k: Tensor, v: Tensor, pos: Tensor, dim_k: int, dim_u: int, num_heads: int,
                       r: Optional[int]) -> Tensor:
    """The formulation of the reference: the local position lambda as a conv3d that builds the B x dim_k x dim_v x H x W
    tensor, then contracted with the queries. Used as the eager baseline of tools/lambda_bench.py."""
    if r is None:
        return lambda_core(q, k, v, pos, dim_k, dim_u, num_heads, r)
    b, _, h, w = q.shape
    n = h * w
    u = dim_u
    dv = v.shape[1] // u
    qh = q.reshape(b, num_heads, dim_k, n)
    sig = k.reshape(b, dim_k, u, n).softmax(-1)
    vu = v.reshape(b, dv, u, n).transpose(1, 2)                              # [b, u, dv, n]
    lc = torch.einsum("bkum,bumv->bkv", sig, vu.transpose(2, 3))
    lp = F.conv3d(vu.reshape(b, u, dv, h, w), pos, padding=(0, r // 2, r // 2)).reshape(b, dim_k, dv, n)
    y = torch.einsum("bhkn,bkvn->bhvn", qh, lp + lc.unsqueeze(-1))
    return y.reshape(b, num_heads * dv, h, w)


def projections(x: Tensor, module, training: bool, dtype=None):
    """(q, k, v) of ``module`` (a LambdaLayer, ours or the reference's) on ``x``: the three 1x1 convolutions and the two
    BatchNorms (batch statistics when ``training``; the running statistics are neither read nor updated then)."""
    dt = x.dtype if dtype is None else dtype

    def bn(t, m):
        if training:
            return F.batch_norm(t, None, None, m.weight.to(dt), m.bias.to(dt), True, 0.0, m.eps)
        return F.batch_norm(t, m.running_mean.to(dt), m.running_var.to(dt), m.weight.to(dt), m.bias.to(dt), False, 0.0,
                            m.eps)

    q = bn(F.conv2d(x, module.to_q.weight.to(dt)), module.norm_q)
    k = F.conv2d(x, module.to_k.weight.to(dt))
    v = bn(F.conv2d(x, module.to_v.weight.to(dt)), module.norm_v)
    return q, k, v


def module_dims(module):
    u = module.u
    dim_k = module.to_k.out_channels // u
    r = module.R.shape[-1] if module.local_contexts else None
    return dim_k, u, module.num_heads, r


def lambda_module(x: Tensor, module, training: bool = True, dtype=None, core=lambda_core) -> Tensor:
    """The reference forward of ``module`` on ``x`` with the parameters cast to ``dtype`` (default: x's)."""
    dt = x.dtype if dtype is None else dtype
    q, k, v = projections(x, module, training, dt)
    dim_k, u, heads, r = module_dims(module)
    pos = (module.R if module.local_contexts else module.pos_emb).to(dt)
    return core(q, k, v, pos, dim_k, u, heads, r)
