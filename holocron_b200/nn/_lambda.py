"""Lambda layer autograd binding (holocron_b200/csrc/lambda_layer.cu) - the key softmax, the content and position lambdas
and their contraction with the queries of the reference's ``LambdaLayer.forward`` (holocron/nn/modules/lambda_layer.py:
70-108), without the B x dim_k x dim_v x H x W position lambda of the local variant."""
from typing import Optional

import torch
from torch import Tensor

from .._lib import check, lib, ptr, require_cuda, stream_ptr
from . import _fused as K

SUPPORTED_DIM_K = (8, 16, 32)
MAX_DIM_U = 4
MAX_HEADS = 8
MAX_R = 23


def check_lambda(dim_k: int, dim_u: int, num_heads: int, r: Optional[int]) -> None:
    """Raises NotImplementedError for the configurations the kernels do not cover."""
    if dim_k not in SUPPORTED_DIM_K:
        raise NotImplementedError(f"LambdaLayer: dim_k {dim_k} (supported: {SUPPORTED_DIM_K})")
    if not 1 <= dim_u <= MAX_DIM_U:
        raise NotImplementedError(f"LambdaLayer: dim_u {dim_u} (supported: 1 to {MAX_DIM_U})")
    if not 1 <= num_heads <= MAX_HEADS:
        raise NotImplementedError(f"LambdaLayer: num_heads {num_heads} (supported: 1 to {MAX_HEADS})")
    if r is not None and r > MAX_R:
        raise NotImplementedError(f"LambdaLayer: r {r} (supported: odd values up to {MAX_R})")


def _v_matrix(v: Tensor, dv: int, u: int, dtype=torch.float32) -> Tensor:
    """v [B, Cvp, H, W] (channel v*u+u') -> [(m, u'), (b, v)], the right operand of the global position lambda."""
    b, _, h, w = v.shape
    vm = v.permute(0, 2, 3, 1).reshape(b, h * w, -1)[:, :, :dv * u].reshape(b, h * w, dv, u)
    return vm.permute(1, 3, 0, 2).reshape(h * w * u, b * dv).to(dtype)


def _pos_matrix(pos_emb: Tensor, dtype=torch.float32) -> Tensor:
    """pos_emb [n, m, k, u] -> [(n, k), (m, u)]."""
    n, m, dk, u = pos_emb.shape
    return pos_emb.detach().to(dtype).permute(0, 2, 1, 3).reshape(n * dk, m * u)


def _global_lp(pm: Tensor, vm: Tensor, b: int, n: int, dk: int, dv: int) -> Tensor:
    """lp[b, n, k, v] = sum_{m,u} pos_emb[n, m, k, u] * v[b, u, v, m], one fp32 GEMM."""
    return (pm @ vm).view(n, dk, b, dv).permute(2, 0, 1, 3).contiguous()


class _LambdaFn(torch.autograd.Function):
    """y = lambda(q, k, v; R or pos_emb): q [B, Cqp, H, W], k [B, Ckp, H, W], v [B, Cvp, H, W] bf16 channels_last with
    zero padding channels (the projections and BatchNorms), R [dk, u, 1, r, r] or pos_emb [n, n, dk, u] fp32 -> y
    [B, heads*dv, H, W] bf16. Saves q, k, v, the softmax statistics and the content lambda; the local variant never
    materialises the position lambda and the global one recomputes its fp32 GEMM in the backward pass for dq only,
    releasing it before the bf16 GEMMs of dv's and pos_emb's shares."""

    @staticmethod
    def forward(ctx, q: Tensor, k: Tensor, v: Tensor, pos: Tensor, dk: int, u: int, heads: int, dv: int, r: int) -> Tensor:
        b, cqp, h, w = q.shape
        ckp, cvp = k.shape[1], v.shape[1]
        cop = K.round_up(heads * dv, 8)
        geom = (b, h, w, dk, u, heads, dv, r, cqp, ckp, cvp, cop)
        dev = q.device
        L = lib()
        stats = torch.empty((b, dk * u, 2), device=dev, dtype=torch.float32)
        lc = torch.empty((b, dk, dv), device=dev, dtype=torch.float32)
        check(L.hb_lambda_content_fwd_bf16(ptr(k), ptr(v), ptr(stats), ptr(lc), *geom, stream_ptr()),
              "hb_lambda_content_fwd_bf16")
        rt = lp = None
        if r:
            rt = pos.detach().float().reshape(dk, u, r * r).permute(2, 1, 0).contiguous()
        else:
            lp = _global_lp(_pos_matrix(pos), _v_matrix(v, dv, u), b, h * w, dk, dv)
        y = K._empty_cl(b, cop, h, w, dev)
        check(L.hb_lambda_out_fwd_bf16(ptr(q), ptr(v), ptr(rt), ptr(lc), ptr(lp), ptr(y), *geom, stream_ptr()),
              "hb_lambda_out_fwd_bf16")
        ctx.save_for_backward(q, k, v, pos, stats, lc)
        ctx.geom = geom
        if cop == heads * dv:
            return y
        # a real allocation, not a view of the padded output: later in-place ops (activations, DropBlock) must work on it
        return y[:, :heads * dv].contiguous(memory_format=torch.channels_last)

    @staticmethod
    def backward(ctx, dy: Tensor):
        q, k, v, pos, stats, lc = ctx.saved_tensors
        geom = ctx.geom
        b, h, w, dk, u, heads, dv, r, cqp, ckp, cvp, cop = geom
        dev = q.device
        L = lib()
        dyb = K.to_channels_last_bf16(dy, cop)
        dlc = torch.empty((b, dk, dv), device=dev, dtype=torch.float32)
        dkt = K._empty_cl(b, ckp, h, w, dev)
        check(L.hb_lambda_bwd_content_bf16(ptr(q), ptr(k), ptr(v), ptr(dyb), ptr(stats), ptr(dlc), ptr(dkt), *geom,
                                           stream_ptr()), "hb_lambda_bwd_content_bf16")
        dvp = K.round_up(dv, 8)
        dlp = torch.empty((b, h * w, dk, dvp), device=dev, dtype=torch.bfloat16)
        check(L.hb_lambda_dlp_bf16(ptr(q), ptr(dyb), ptr(dlp), *geom, stream_ptr()), "hb_lambda_dlp_bf16")
        rt = lp = dvpos = dpos = None
        if r:
            rt = pos.detach().float().reshape(dk, u, r * r).permute(2, 1, 0).contiguous()
        else:
            lp = _global_lp(_pos_matrix(pos), _v_matrix(v, dv, u), b, h * w, dk, dv)
        dq = K._empty_cl(b, cqp, h, w, dev)
        check(L.hb_lambda_bwd_q_bf16(ptr(dyb), ptr(v), ptr(rt), ptr(lc), ptr(lp), ptr(dq), *geom, stream_ptr()),
              "hb_lambda_bwd_q_bf16")
        lp = None   # the recomputed fp32 position lambda is released before the gradient GEMMs allocate
        if not r:
            # dv's and pos_emb's shares of the position lambda: two GEMMs over the bf16 dlp (fp32 accumulation)
            n = h * w
            dm = dlp[..., :dv].permute(1, 2, 0, 3).reshape(n * dk, b * dv)
            dvpos = (_pos_matrix(pos, torch.bfloat16).t() @ dm).view(n, u, b, dv).permute(2, 0, 3, 1)
            dvpos = dvpos.reshape(b, n, dv * u).float().contiguous()   # with u = 1 the reshape is a strided view
            if ctx.needs_input_grad[3]:
                dpos = (dm @ _v_matrix(v, dv, u, torch.bfloat16).t()).view(n, dk, n, u).permute(0, 2, 1, 3).to(pos.dtype)
            del dm
        dvo = K._empty_cl(b, cvp, h, w, dev)
        check(L.hb_lambda_bwd_v_bf16(ptr(k), ptr(stats), ptr(dlc), ptr(dlp), ptr(rt), ptr(dvpos), ptr(dvo), *geom,
                                     stream_ptr()), "hb_lambda_bwd_v_bf16")
        if r and ctx.needs_input_grad[3]:
            scratch = torch.empty(b * dk * u * r * r, device=dev, dtype=torch.float32)
            dr = torch.empty((dk, u, 1, r, r), device=dev, dtype=torch.float32)
            check(L.hb_lambda_bwd_r_bf16(ptr(dlp), ptr(v), ptr(scratch), ptr(dr), *geom, stream_ptr()),
                  "hb_lambda_bwd_r_bf16")
            dpos = dr.to(pos.dtype)
        return dq, dkt, dvo, dpos, None, None, None, None, None


def lambda_layer(q: Tensor, k: Tensor, v: Tensor, pos: Tensor, dim_k: int, dim_u: int, num_heads: int, dim_v: int,
                 r: Optional[int]) -> Tensor:
    """The lambda of ``q`` (channel h*dim_k+k), ``k`` (k*dim_u+u) and ``v`` (v*dim_u+u), bf16 channels_last tensors whose
    widths are the logical channels zero-padded to a multiple of 8, with the local embedding ``R`` (``r`` odd) or the
    global ``pos_emb`` (``r`` None); returns bf16 [B, num_heads*dim_v, H, W] (channel h*dim_v+v)."""
    require_cuda(q, k, v, pos)
    check_lambda(dim_k, dim_u, num_heads, r)
    b, _, h, w = q.shape
    if r is None and pos.shape[0] * pos.shape[1] != (h * w) ** 2:
        raise RuntimeError(f"LambdaLayer: {h}x{w} = {h * w} positions, the positional embedding holds {pos.shape[0]}")
    for t, c in ((q, num_heads * dim_k), (k, dim_k * dim_u), (v, dim_v * dim_u)):
        if t.shape[0] != b or tuple(t.shape[2:]) != (h, w) or t.shape[1] < c or t.shape[1] % 8:
            raise RuntimeError(f"LambdaLayer: projection of shape {tuple(t.shape)}, expected >= {c} channels")
    qb, kb, vb = (K.to_channels_last_bf16(t) for t in (q, k, v))
    return _LambdaFn.apply(qb, kb, vb, pos, int(dim_k), int(dim_u), int(num_heads), int(dim_v), int(r or 0))
