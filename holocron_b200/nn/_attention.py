"""Attention autograd bindings (holocron_b200/csrc/attention.cu): the reference's ``SAM`` (x * sigmoid(conv1x1(x)),
holocron/nn/modules/attention.py:17-30) and the ``DimAttention`` branches of ``TripletAttention`` (:33-77) without the
transposed copies, the separate z_pool / convolution / BatchNorm / sigmoid passes or the broadcast products.

bf16 and fp32 tensors run natively; other float dtypes are computed in fp32 and cast back. Outputs are channels_last with
the channel pitch rounded up to one 16-byte vector (the padding channels never feed a result and are cropped here).
Gates, pooled planes, statistics and parameter gradients are fp32."""
import ctypes
from typing import List, Optional, Sequence, Tuple

import torch
from torch import Tensor, nn

from .._lib import check, dtype_code, lib, ptr, require_cuda, stream_ptr
from ._fused import BNBranch, _bn_batch_stats, _empty_cl, attach_stats, sync_group
from ._nhwc import compute_dtype, crop, nhwc, pitch, require_4d, run_native

_VP3 = ctypes.c_void_p * 3
_I3 = ctypes.c_int * 3
_TAPS = 2 * 7 * 7
SAM_MAX_VECTORS = 128   # channel vectors of 16 bytes per pixel row the SAM backward kernel holds in registers
_THREADS = 256   # elements per CTA of the plane kernels: one partial row each


def _vp3(ts: Sequence[Optional[Tensor]]):
    return _VP3(*[0 if t is None else t.data_ptr() for t in ts])


def _f32(t: Tensor) -> Tensor:
    return t.detach().reshape(-1).float().contiguous()


def _enabled(en: Sequence[bool], make) -> List[Optional[Tensor]]:
    """make(b) for each enabled branch b, None for the others."""
    return [make(b) if en[b] else None for b in range(3)]


# --------------------------------------------------------------------------------------------------------- SAM
class _SamFn(torch.autograd.Function):
    """x [N, C, H, W] -> y [N, Cp, H, W] channels_last (the caller drops the padding channels)."""

    @staticmethod
    def forward(ctx, x: Tensor, weight: Tensor, bias: Tensor) -> Tensor:
        n, c, h, w = x.shape
        cp = pitch(c, x.dtype)
        xc = nhwc(x, cp)
        w32, b32 = _f32(weight), _f32(bias)
        y = _empty_cl(n, cp, h, w, xc.device, xc.dtype)
        gate = torch.empty(n * h * w, dtype=torch.float32, device=x.device)
        check(lib().hb_sam_fwd(ptr(xc), ptr(w32), ptr(b32), ptr(y), ptr(gate), n * h * w, c, cp, dtype_code(xc),
                               stream_ptr()), "hb_sam_fwd")
        ctx.save_for_backward(xc, w32, gate)
        ctx.cfg = (c, weight.dtype, weight.shape, bias.dtype)
        return y

    @staticmethod
    def backward(ctx, dy: Tensor):
        xc, w32, gate = ctx.saved_tensors
        c, wdt, wshape, bdt = ctx.cfg
        n, cp, h, w = xc.shape
        dyc = dy.contiguous(memory_format=torch.channels_last)
        L = lib()
        dt = dtype_code(xc)
        slots = L.hb_sam_bwd_slots(n * h * w, c, cp, dt)
        part = torch.empty((max(slots, 1), cp + 1), dtype=torch.float32, device=xc.device)
        dwdb = torch.empty(c + 1, dtype=torch.float32, device=xc.device)
        dx = _empty_cl(n, cp, h, w, xc.device, xc.dtype)
        check(L.hb_sam_bwd(ptr(xc), ptr(dyc), ptr(w32), ptr(gate), ptr(dx), ptr(part), ptr(dwdb), n * h * w, c, cp, dt,
                           stream_ptr()), "hb_sam_bwd")
        return crop(dx, c), dwdb[:c].view(wshape).to(wdt), dwdb[c:].to(bdt)


def sam(x: Tensor, weight: Tensor, bias: Tensor) -> Tensor:
    """SAM's forward (reference attention.py:29-30): x * sigmoid(conv2d(x, weight, bias)) with a [1, C, 1, 1] filter."""
    require_4d("SAM", x)
    if x.shape[1] != weight.shape[1]:
        raise RuntimeError(f"SAM: built for {weight.shape[1]} channels, got an input with {x.shape[1]}")
    dt = compute_dtype(x.dtype)
    if pitch(x.shape[1], dt) * dt.itemsize > 16 * SAM_MAX_VECTORS:
        raise NotImplementedError(f"SAM: at most {16 * SAM_MAX_VECTORS // dt.itemsize} channels in {dt}, got "
                                  f"{x.shape[1]}")
    require_cuda(x)
    return run_native(_SamFn, x, weight, bias)


# --------------------------------------------------------------------------------------------------------- triplet
# branch b of TripletAttention reduces dim b + 1 of x [N, C, H, W]; its z_pool plane is rows x cols:
#   C branch (dim 1): H x W, H branch (dim 2): C x W, W branch (dim 3): H x C
def _plane_dims(b: int, c: int, h: int, w: int) -> Tuple[int, int]:
    return ((h, w), (c, w), (h, c))[b]


def _uses_batch_stats(bn: nn.BatchNorm2d) -> bool:
    """What F.batch_norm does with the module's flags: batch statistics in training or without running statistics."""
    return bn.training or bn.running_mean is None


class _TripletFn(torch.autograd.Function):
    """x [N, C, H, W] -> y [N, Cp, H, W] channels_last over the enabled branches (the caller drops the padding
    channels). ``bns``: the BatchNorm2d of each branch or None; the parameters follow in branch order, conv weight,
    BatchNorm weight and bias of each (None for a disabled branch)."""

    @staticmethod
    def forward(ctx, x: Tensor, bns, *params) -> Tensor:
        n, c, h, w = x.shape
        cp = pitch(c, x.dtype)
        dev = x.device
        xc = nhwc(x, cp)
        L = lib()
        dt = dtype_code(xc)
        en = [bn is not None for bn in bns]
        dims = [_plane_dims(b, c, h, w) for b in range(3)]
        f32 = dict(dtype=torch.float32, device=dev)
        planes = _enabled(en, lambda b: torch.empty((n, 2) + dims[b], **f32))
        idx = _enabled(en, lambda b: torch.empty((n,) + dims[b], dtype=torch.int32, device=dev))
        hp = [None, None, None]
        if en[1]:
            nhb = -(-h // L.hb_triplet_row_block(h, c, cp, dt))
            hp = [torch.empty((n, nhb, w, c), **f32), torch.empty((n, nhb, w, c), **f32),
                  torch.empty((n, nhb, w, c), dtype=torch.int32, device=dev)]
        check(L.hb_triplet_pool_fwd(ptr(xc), ptr(planes[0]), ptr(idx[0]), ptr(planes[2]), ptr(idx[2]), ptr(hp[0]),
                                    ptr(hp[1]), ptr(hp[2]), ptr(planes[1]), ptr(idx[1]), n, h, w, c, cp, dt,
                                    stream_ptr()), "hb_triplet_pool_fwd")
        rows = _I3(*[d[0] for d in dims])
        cols = _I3(*[d[1] for d in dims])
        blocks = [-(-(n * d[0] * d[1]) // _THREADS) for d in dims]
        wts = _enabled(en, lambda b: _f32(params[3 * b]))
        z = _enabled(en, lambda b: torch.empty((n, 1) + dims[b], **f32))
        parts = _enabled(en, lambda b: torch.empty((blocks[b], 1, 2), **f32))
        slots = _I3()
        check(L.hb_triplet_conv_fwd(_vp3(planes), _vp3(wts), _vp3(z), _vp3(parts), slots, rows, cols, n,
                                    stream_ptr()), "hb_triplet_conv_fwd")
        stats = _enabled(en, lambda b: torch.empty((4, 1), **f32))
        train = None
        for b in range(3):
            if not en[b]:
                continue
            bn = bns[b]
            g32 = _f32(params[3 * b + 1]) if params[3 * b + 1] is not None else None
            b32 = _f32(params[3 * b + 2]) if params[3 * b + 2] is not None else None
            if _uses_batch_stats(bn):
                attach_stats(z[b], parts[b], slots[b])
                _bn_batch_stats([z[b]], [BNBranch(bn)], [g32], [b32], stats[b], 1, 1, n * dims[b][0] * dims[b][1])
            else:
                check(L.hb_bn_eval_affine(ptr(g32), ptr(b32), ptr(bn.running_mean), ptr(bn.running_var),
                                          ctypes.c_float(bn.eps), 1, 1, ptr(stats[b][2]), ptr(stats[b][3]),
                                          ptr(stats[b][0]), ptr(stats[b][1]), stream_ptr()), "hb_bn_eval_affine")
            train = _uses_batch_stats(bn)
        gates = _enabled(en, lambda b: torch.empty((n,) + dims[b], **f32))
        check(L.hb_triplet_gate(_vp3(z), _vp3(stats), _vp3(gates), rows, cols, n, stream_ptr()), "hb_triplet_gate")
        y = _empty_cl(n, cp, h, w, dev, xc.dtype)
        check(L.hb_triplet_apply(ptr(xc), ptr(y), ptr(gates[0]), ptr(gates[1]), ptr(gates[2]), n, h, w, c, cp, dt,
                                 stream_ptr()), "hb_triplet_apply")
        ctx.save_for_backward(xc, *planes, *idx, *z, *gates, *stats, *wts)
        ctx.cfg = (en, c, blocks, [p.dtype if p is not None else None for p in params],
                   [p.shape if p is not None else None for p in params], bool(train))
        return y

    @staticmethod
    def backward(ctx, dy: Tensor):
        xc, *saved = ctx.saved_tensors
        planes, idx, z, gates, stats, wts = (saved[3 * k:3 * k + 3] for k in range(6))
        en, c, blocks, pdt, pshape, train = ctx.cfg
        n, cp, h, w = xc.shape
        dev = xc.device
        L = lib()
        dt = dtype_code(xc)
        dims = [_plane_dims(b, c, h, w) for b in range(3)]
        rows = _I3(*[d[0] for d in dims])
        cols = _I3(*[d[1] for d in dims])
        f32 = dict(dtype=torch.float32, device=dev)
        dyc = dy.contiguous(memory_format=torch.channels_last)
        dg = _enabled(en, lambda b: torch.empty((n,) + dims[b], **f32))
        hp_sum = None
        if en[1]:
            hp_sum = torch.empty((n, -(-h // L.hb_triplet_row_block(h, c, cp, dt)), w, c), **f32)
        check(L.hb_triplet_pool_bwd(ptr(xc), ptr(dyc), ptr(dg[0]), ptr(dg[2]), ptr(hp_sum), ptr(dg[1]), n, h, w, c,
                                    cp, dt, stream_ptr()), "hb_triplet_pool_bwd")
        dz = _enabled(en, lambda b: torch.empty((n,) + dims[b], **f32))
        bparts = _enabled(en, lambda b: torch.empty((blocks[b], 2), **f32))
        dgamma = _enabled(en, lambda b: torch.empty(1, **f32))
        dbeta = _enabled(en, lambda b: torch.empty(1, **f32))
        check(L.hb_triplet_bn_bwd(_vp3(dg), _vp3(z), _vp3(gates), _vp3(stats), _vp3(dz), _vp3(bparts),
                                  _vp3(dgamma), _vp3(dbeta), rows, cols, n, ctypes.c_float(1.0 / sum(en)),
                                  int(train), stream_ptr()), "hb_triplet_bn_bwd")
        dplane = _enabled(en, lambda b: torch.empty((n, 2) + dims[b], **f32))
        wparts = _enabled(en, lambda b: torch.empty((blocks[b], _TAPS), **f32))
        dw = _enabled(en, lambda b: torch.empty(_TAPS, **f32))
        check(L.hb_triplet_conv_bwd(_vp3(planes), _vp3(wts), _vp3(dz), _vp3(dplane), _vp3(wparts), _vp3(dw), rows,
                                    cols, n, stream_ptr()), "hb_triplet_conv_bwd")
        dx = _empty_cl(n, cp, h, w, dev, xc.dtype)
        check(L.hb_triplet_dx(ptr(dyc), ptr(dx), ptr(gates[0]), ptr(gates[1]), ptr(gates[2]), ptr(dplane[0]),
                              ptr(dplane[1]), ptr(dplane[2]), ptr(idx[0]), ptr(idx[1]), ptr(idx[2]), n, h, w, c, cp,
                              dt, stream_ptr()), "hb_triplet_dx")
        grads: List[Optional[Tensor]] = []
        for b in range(3):
            for k, g in enumerate((dw[b], dgamma[b], dbeta[b])):
                i = 3 * b + k
                grads.append(None if g is None or pdt[i] is None else g.view(pshape[i]).to(pdt[i]))
        return crop(dx, c), None, *grads


def triplet_attention(x: Tensor, branches: Sequence[Tuple[int, nn.Conv2d, nn.BatchNorm2d]]) -> Tensor:
    """The mean over ``branches`` of x gated along each branch's dim (DimAttention.forward, attention.py:50-56, and
    TripletAttention.forward, :72-77). A branch is (dim, 7x7 conv, BatchNorm2d) with dim in 1..3 or its negative form;
    one launch sequence serves every branch."""
    require_4d("TripletAttention", x)
    n, c, h, w = x.shape
    bns: List[Optional[nn.BatchNorm2d]] = [None, None, None]
    params: List[Optional[Tensor]] = [None] * 9
    for dim, conv, bn in branches:
        if dim not in (1, 2, 3, -1, -2, -3):
            raise NotImplementedError(f"DimAttention: dim in 1..3 (or its negative form) only, got {dim}")
        b = dim % 4 - 1
        if bns[b] is not None:
            raise NotImplementedError(f"TripletAttention: two branches attend over dim {b + 1}")
        if sync_group([bn], bn.training) is not None:
            # the gate kernels keep each branch's statistics on the device between their launches: no all-reduce point
            raise NotImplementedError("TripletAttention: a SyncBatchNorm that synchronises over its process group "
                                      "(its statistics would silently stay per-GPU)")
        rows, cols = _plane_dims(b, c, h, w)
        if _uses_batch_stats(bn) and n * rows * cols == 1:   # F.batch_norm's check, before any launch
            raise ValueError(f"Expected more than 1 value per channel when training, got input size "
                             f"{torch.Size((n, 1, rows, cols))}")
        bns[b] = bn
        params[3 * b:3 * b + 3] = [conv.weight, bn.weight, bn.bias]
    if pitch(c, compute_dtype(x.dtype)) > 2048:
        raise NotImplementedError(f"TripletAttention: at most 2048 channels, got {c}")
    if len({_uses_batch_stats(bn) for bn in bns if bn is not None}) > 1:
        raise NotImplementedError("TripletAttention: branches mixing training and evaluation BatchNorm modes")
    require_cuda(x)
    return run_native(_TripletFn, x, tuple(bns), *params)
