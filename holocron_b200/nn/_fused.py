"""Autograd bindings of the tensor-core convolution and the fused BatchNorm/branch-sum/activation kernels.

Activations travel between these ops as NCHW-logical ``bfloat16`` tensors in ``torch.channels_last`` memory format
(physically NHWC, which is what the TMA descriptors of the kernels address). Parameters stay fp32 with the
reference's shapes (``Cout x Cin x kh x kw``) so ``state_dict`` is interchangeable with the reference's modules.

Reference call sites being replaced: ``nn.Conv2d`` / ``nn.BatchNorm2d`` / activation modules emitted by
``holocron.models.utils.conv_sequence`` (holocron/models/utils.py:28-86) and ``RepBlock.forward``
(holocron/models/classification/repvgg.py:71-73).
"""
import ctypes
import functools
import os
import weakref
from typing import List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist
from torch import Tensor, nn

from .._lib import DTYPE_CODE, ConvArgs, check, dtype_code, lib, ptr, require_cuda, stream_ptr

ACT_NONE, ACT_RELU, ACT_RELU6, ACT_SILU, ACT_LEAKY, ACT_MISH, ACT_HARDMISH, ACT_FRELU = range(8)

_c_float = ctypes.c_float
_VP3 = ctypes.c_void_p * 3

# Optional per-launch timing (bench.py's roofline leg): when set to a list, every launch that ACTUALLY happened (return
# code 0) appends (kind, info, start_event, end_event) recorded on the launching stream. ``info`` carries the algorithmic
# work of that launch (SURVEY.md §8d): ``flops`` and ``bytes``.
KERNEL_TIMER = None


def _timed(kind: str, info: dict, fn):
    """Runs ``fn`` (returns a C-ABI return code); records the event pair only when a kernel was launched (rc == 0)."""
    if KERNEL_TIMER is None:
        return fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    rc = fn()
    e1.record()
    if rc == 0:
        KERNEL_TIMER.append((kind, info, e0, e1))
    return rc


def conv_work(m_out: int, cout: int, k_total: int, in_elems: int, w_elems: int, out_elems: Optional[int] = None,
              w_bytes_per: int = 2) -> dict:
    """Algorithmic work of one dense convolution launch: 2*M*Cout*K FLOPs (K = sum over taps/sources of the channels
    actually multiplied); bytes = activations read + written (bf16) + filter bytes."""
    out_elems = m_out * cout if out_elems is None else out_elems
    return {"flops": 2.0 * m_out * cout * k_total, "bytes": 2.0 * (in_elems + out_elems) + w_bytes_per * w_elems}


# ---- column statistics travelling with a tensor (training-mode BatchNorm without a statistics pass) ----
@functools.lru_cache(maxsize=None)
def _sm_count(index: int) -> int:
    return torch.cuda.get_device_properties(index).multi_processor_count


def conv_stat_slots(device) -> int:
    """Statistics slots of a convolution epilogue: 2 consumer warpgroups x (<= one CTA per SM)."""
    return 2 * _sm_count(torch.device(device).index or 0)


def bn_stat_slots(device) -> int:
    """Statistics slots of the streaming BatchNorm kernels: <= 4 blocks per SM."""
    return 4 * _sm_count(torch.device(device).index or 0)


def epilogue_stats_pay_off(k_total: int) -> bool:
    """Whether the convolution epilogue should also produce the BatchNorm statistics of its output. The extra
    shared-memory pass over the staged tile is cheap next to the main loop only where the tile time is set by the tensor
    pipe (K = R*S*Cin large); on the narrow layers (48 .. 96 channels) it lengthens the epilogue, which the consumer
    warpgroups run after their MMAs. The K >= 1024 threshold has not been re-tuned on the H100.
    HB_FORCE_CONV_STATS / HB_DISABLE_CONV_STATS override."""
    if os.environ.get("HB_DISABLE_CONV_STATS"):
        return False
    if os.environ.get("HB_FORCE_CONV_STATS"):
        return True
    return k_total >= 1024


def attach_stats(t: Tensor, parts: Tensor, slots: int) -> None:
    """Marks ``t`` ([N, C, H, W] bf16 NHWC) as carrying per-channel (sum, sum of squares) partials ``parts`` [cap, C, 2]."""
    t._hb_stats = (parts, int(slots), t._version)


def get_stats(t: Tensor):
    st = getattr(t, "_hb_stats", None)
    if st is None or st[2] != t._version or st[0].shape[1] != t.shape[1] or st[1] < 1:
        return None
    return st[0], st[1]


def direct_grad(p: Tensor, krsc: bool = False) -> Optional[Tensor]:
    """The parameter's gradient buffer when the backward kernels may ADD into it themselves (opt-in per parameter through
    ``_hb_direct_grad``, set by :class:`holocron_b200.distributed.GradBucket`): fp32, the parameter's shape, and - for
    filters - physically KRSC. Autograd then receives ``None`` for this parameter (no AccumulateGrad kernel)."""
    if not getattr(p, "_hb_direct_grad", False):
        return None
    g = p.grad
    if g is None or g.dtype != torch.float32 or g.shape != p.shape or not g.is_cuda:
        return None
    if krsc:
        if g.ndim != 4 or not g.permute(0, 2, 3, 1).is_contiguous():
            return None
    elif not g.is_contiguous():
        return None
    return g


def act_code(act: Optional[nn.Module]) -> Tuple[int, float]:
    """Maps an activation module instance to the kernels' activation code (+ negative slope)."""
    if act is None or isinstance(act, nn.Identity):
        return ACT_NONE, 0.0
    if isinstance(act, nn.ReLU6):
        return ACT_RELU6, 0.0
    if isinstance(act, nn.ReLU):
        return ACT_RELU, 0.0
    if isinstance(act, nn.SiLU):
        return ACT_SILU, 0.0
    if isinstance(act, nn.LeakyReLU):
        return ACT_LEAKY, float(act.negative_slope)
    if isinstance(act, nn.Mish):
        return ACT_MISH, 0.0
    if type(act).__name__ == "HardMish":
        return ACT_HARDMISH, 0.0
    raise NotImplementedError(f"no fused kernel for activation {type(act).__name__}")


def round_up(v: int, m: int) -> int:
    return (v + m - 1) // m * m


def to_channels_last_bf16(x: Tensor, c_pad: Optional[int] = None) -> Tensor:
    """NCHW-logical tensor of any float dtype / layout -> bf16 channels_last, channels optionally zero-padded.
    Already-conforming tensors are returned as is (no copy)."""
    require_cuda(x)
    n, c, h, w = x.shape
    cp = c if c_pad is None else c_pad
    if cp == c and x.dtype == torch.bfloat16 and x.is_contiguous(memory_format=torch.channels_last):
        return x
    no_grad = not (x.requires_grad and torch.is_grad_enabled())   # the raw kernel is invisible to autograd
    if no_grad and x.is_contiguous() and x.dtype in (torch.float32, torch.bfloat16, torch.float16) and (cp != c or c < 8):
        out = torch.empty((n, cp, h, w), device=x.device, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
        check(lib().hb_nchw_to_nhwc_pad_bf16(ptr(x), ptr(out), n, c, h, w, cp, dtype_code(x), stream_ptr()),
              "hb_nchw_to_nhwc_pad_bf16")
        return out
    y = x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    if cp != c:
        out = torch.zeros((n, cp, h, w), device=x.device, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
        out[:, :c] = y
        return out
    return y


def _empty_cl(n: int, c: int, h: int, w: int, device, dtype=torch.bfloat16) -> Tensor:
    # a real channels_last allocation, not a permuted VIEW: outputs of custom autograd Functions that are views may not be
    # modified in place afterwards (the in-place DropBlock2d that conv_sequence puts behind every activation does that)
    return torch.empty((n, c, h, w), device=device, dtype=dtype, memory_format=torch.channels_last)


# ------------------------------------------------------------------------------------------------------
# filter packing cache: fp32 master (any layout) -> bf16 KRSC for fprop, flipped+transposed bf16 for dgrad
class PackedFilter:
    __slots__ = ("wf", "wd", "key", "cin_p", "cout_p", "cin_d", "cout", "cin", "r", "s", "wref", "w_krsc", "need_dgrad")


_pack_cache = {}


class _PackTable:
    """Device table of every registered filter, so that ONE launch (hb_pack_conv_weights_multi) re-packs the whole
    network when the optimizer has changed the parameters (all of them change every step) instead of one launch per
    layer. Filters join the table the first time they are packed; the table is rebuilt only when its membership or a
    pointer changes, so under CUDA-graph capture the multi-tensor launch is the only packing work in the graph."""

    def __init__(self) -> None:
        self.sig = None
        self.metas = None
        self.chunks = None
        self.num_chunks = 0

    def repack_all(self) -> bool:
        ents = []
        for k, e in list(_pack_cache.items()):
            w = e.wref()
            if w is None:
                del _pack_cache[k]
                continue
            if e.w_krsc is None:          # non-channels_last master: needs its own permuted copy, packed individually
                continue
            if e.w_krsc.data_ptr() != w.data_ptr():   # the parameter moved to new storage: its view here is stale
                del _pack_cache[k]
                continue
            ents.append((e, w))
        if len(ents) < 2:
            return False
        sig = tuple((e.w_krsc.data_ptr(), e.wf.data_ptr(), 0 if e.wd is None else e.wd.data_ptr()) for e, _ in ents)
        L = lib()
        if sig != self.sig:
            import numpy as np
            chunk = L.hb_pack_chunk_elems()
            dt = np.dtype([("ptrs", "<u8", (3,)), ("ints", "<i4", (8,))])
            assert dt.itemsize == L.hb_pack_meta_bytes()
            metas = np.zeros(len(ents), dtype=dt)
            rows = []
            for i, (e, _) in enumerate(ents):
                metas[i]["ptrs"] = sig[i]
                metas[i]["ints"] = (e.cout, e.cin, e.r, e.s, e.cin_p, e.cin_d, e.cout_p, e.cout_p)
                n = e.wf.numel() + (0 if e.wd is None else e.wd.numel())
                nch = (n + chunk - 1) // chunk
                rows.append(np.stack([np.full(nch, i, dtype=np.int32), np.arange(nch, dtype=np.int32)], 1))
            chunks = np.ascontiguousarray(np.concatenate(rows, 0))
            dev = ents[0][0].wf.device
            self.metas = torch.from_numpy(metas.view(np.uint8).reshape(len(ents), -1).copy()).to(dev)
            self.chunks = torch.from_numpy(chunks).to(dev)
            self.num_chunks = int(chunks.shape[0])
            self.sig = sig
        check(L.hb_pack_conv_weights_multi(ptr(self.metas), ptr(self.chunks), self.num_chunks, stream_ptr()),
              "hb_pack_conv_weights_multi")
        for e, w in ents:
            e.key = (w.data_ptr(), w._version, e.need_dgrad, tuple(w.stride()), e.cin_p, tuple(w.shape))
        return True


_pack_table = _PackTable()


def pack_filter(weight: Tensor, need_dgrad: bool, cin_p: Optional[int] = None) -> PackedFilter:
    """bf16 KRSC copy of an fp32 (Cout, Cin, kh, kw) filter, rows zero-padded to Cout % 16 == 0 and channels to
    ``cin_p`` (the channel count of the activation it will meet, >= Cin, % 8 == 0); plus, for the data-gradient pass,
    the flipped/transposed filter [cin_d][R][S][cout_p] with cin_d % 16 == 0."""
    cout, cin, r, s = weight.shape
    if cin_p is None:
        cin_p = round_up(cin, 8)
    key = (weight.data_ptr(), weight._version, need_dgrad, tuple(weight.stride()), cin_p, tuple(weight.shape))
    ent = _pack_cache.get(id(weight))
    if ent is not None and ent.wref() is not weight:
        # a dead parameter's id (and possibly its CUDA block and init-time version) recycled by a new one
        del _pack_cache[id(weight)]
        ent = None
    if ent is not None and ent.key == key:
        return ent
    if ent is not None and ent.key[0] == key[0] and ent.key[2:] == key[2:] and ent.wref() is weight and ent.w_krsc is not None:
        # same filter, new parameter values (an optimizer step): refresh every registered filter in one launch
        if _pack_table.repack_all() and ent.key == key:
            return ent
    w = weight.detach()
    if w.dtype != torch.float32:
        w = w.float()
    # physical KRSC fp32 view (zero-copy when the parameter is stored channels_last)
    w_krsc = w.permute(0, 2, 3, 1)
    zero_copy = w_krsc.is_contiguous() and w.dtype == weight.dtype
    if not w_krsc.is_contiguous():
        w_krsc = w_krsc.contiguous()
    ent = PackedFilter()
    ent.key, ent.cin_p, ent.cout, ent.cin, ent.r, ent.s = key, cin_p, cout, cin, r, s
    ent.cout_p = round_up(cout, 16)
    ent.cin_d = round_up(cin_p, 16)
    ent.need_dgrad = need_dgrad
    wid = id(weight)
    ent.wref = weakref.ref(weight, lambda _r, wid=wid: _pack_cache.pop(wid, None) if _pack_cache.get(wid) is not None
                           and _pack_cache[wid].wref() is None else None)
    # only views of a live PARAMETER can sit in the device table: a per-step temporary (ConvNeXt's patchify filters are
    # permuted views rebuilt every forward) would change the table's membership every step - a host->device rebuild that a
    # CUDA-graph capture cannot contain; such filters are packed by their own launch each time
    ent.w_krsc = w_krsc if (zero_copy and isinstance(weight, nn.Parameter)) else None
    ent.wf = torch.empty((ent.cout_p, r, s, cin_p), device=w.device, dtype=torch.bfloat16)
    ent.wd = torch.empty((ent.cin_d, r, s, ent.cout_p), device=w.device, dtype=torch.bfloat16) if need_dgrad else None
    check(lib().hb_pack_conv_weights(ptr(w_krsc), ptr(ent.wf), ptr(ent.wd), cout, cin, r, s, cin_p, ent.cin_d, ent.cout_p,
                                     ent.cout_p, stream_ptr()), "hb_pack_conv_weights")
    _pack_cache[id(weight)] = ent
    return ent


_s2_cache = {}


def dgrad_s2_filters(weight: Tensor, cin_d: int, cout_p: int) -> Tensor:
    """bf16 class filters of the stride-2 3x3 data gradient (hb_pack_dgrad_s2_weights), cached per parameter version."""
    key = (weight.data_ptr(), weight._version, tuple(weight.stride()), cin_d, cout_p, tuple(weight.shape))
    ent = _s2_cache.get(id(weight))
    if ent is not None and ent[0] == key and ent[2]() is weight:
        return ent[1]
    cout, cin = weight.shape[0], weight.shape[1]
    w_krsc = weight.detach().float().permute(0, 2, 3, 1)
    if not w_krsc.is_contiguous():
        w_krsc = w_krsc.contiguous()
    out = torch.empty(9 * cin_d * cout_p, device=weight.device, dtype=torch.bfloat16)
    check(lib().hb_pack_dgrad_s2_weights(ptr(w_krsc), ptr(out), cout, cin, cin_d, cout_p, stream_ptr()),
          "hb_pack_dgrad_s2_weights")
    wid = id(weight)
    _s2_cache[wid] = (key, out, weakref.ref(weight, lambda _r, wid=wid: _s2_cache.pop(wid, None)
                                             if wid in _s2_cache and _s2_cache[wid][2]() is None else None))
    return out


def dgrad_s2_raw(dyb: Tensor, weight: Tensor, cin_d: int, h: int, w: int, dy1: Optional[Tensor] = None,
                 wd1: Optional[Tensor] = None) -> Tensor:
    """dx [N, cin_d, h, w] of a stride-2 3x3 pad-1 convolution from dy [N, cout_p, ho, wo] (+ the 1x1 stride-2 branch
    of a RepVGG block) by parity classes - no zero insertion."""
    n, cout_p, ho, wo = dyb.shape
    dxp = _empty_cl(n, cin_d, h, w, dyb.device)
    wcls = dgrad_s2_filters(weight, cin_d, cout_p)
    # parity classes: (1 + a)(1 + b) taps on the class' pixels = 9/4 taps per dx pixel (+ the 1x1 branch on class (0,0))
    taps = sum((1 + a) * (1 + b) * ((h - a + 1) // 2) * ((w - b + 1) // 2) for a in (0, 1) for b in (0, 1))
    nsrc = 2 if dy1 is not None else 1
    info = dict(shape=("dgrad_s2", h, cout_p, cin_d, 3, 2), launches=4 + (nsrc - 1),
                flops=2.0 * n * cin_d * cout_p * (taps + (nsrc - 1) * ho * wo),
                bytes=2.0 * (nsrc * n * ho * wo * cout_p + n * h * w * cin_d) + 2.0 * (9 + nsrc - 1) * cin_d * cout_p)
    check(_timed("dgrad", info, lambda: lib().hb_conv2d_dgrad_s2_bf16(
        ptr(dyb), ptr(wcls), ptr(dy1), ptr(wd1), ptr(dxp), n, h, w, ho, wo, cout_p, cin_d, 0, stream_ptr())),
        "hb_conv2d_dgrad_s2_bf16")
    return dxp


def _pad_vec(v: Optional[Tensor], n: int) -> Optional[Tensor]:
    if v is None:
        return None
    v = v.detach().float().contiguous()
    if v.numel() == n:
        return v
    out = torch.zeros(n, device=v.device, dtype=torch.float32)
    out[:v.numel()] = v
    return out


def conv_out_size(h: int, k: int, stride: int, pad: int, dil: int) -> int:
    return (h + 2 * pad - dil * (k - 1) - 1) // stride + 1


def conv2d_forward_raw(x: Tensor, wf: Tensor, cout: int, r: int, s: int, stride: int, pad: int, dil: int,
                       bias: Optional[Tensor] = None, residual: Optional[Tensor] = None, act: int = ACT_NONE, *,
                       w2: Optional[Tensor] = None, xe: Optional[Tensor] = None, we: Optional[Tensor] = None,
                       want_stats: bool = False, kind: str = "fprop", norm: Optional[Tuple[Tensor, Tensor, Tensor]] = None):
    """x: bf16 channels_last [N, Cin_p, H, W]; wf: bf16 [Cout, R, S, Cin_p] -> bf16 channels_last [N, Cout, Ho, Wo].

    One launch of ``hb_conv2d_fused_bf16``. ``w2`` ([Cout, 1, 1, Cin_p]): dual output, returns ``(y, y2)`` with
    ``y2 = conv1x1(x, w2)`` (same stride, pad 0) computed from the centre-tap loads. ``xe`` / ``we``: K extension,
    ``y += conv1x1(xe, we)`` in the same accumulator. ``want_stats``: the outputs carry their per-channel statistics
    partials (:func:`get_stats`) for the training-mode BatchNorm that follows."""
    n, cin_p, h, w = x.shape
    ho, wo = conv_out_size(h, r, stride, pad, dil), conv_out_size(w, s, stride, pad, dil)
    y = _empty_cl(n, cout, ho, wo, x.device)
    y2 = _empty_cl(n, cout, ho, wo, x.device) if w2 is not None else None
    a = ConvArgs()
    a.x, a.w, a.y = x.data_ptr(), wf.data_ptr(), y.data_ptr()
    a.bias = 0 if bias is None else bias.data_ptr()
    a.residual = 0 if residual is None else residual.data_ptr()
    a.N, a.H, a.W, a.Cin, a.Cout, a.R, a.S = n, h, w, cin_p, cout, r, s
    a.stride, a.pad, a.dil, a.act, a.num_ctas = stride, pad, dil, act, 0
    m_out = n * ho * wo
    k_total = r * s * cin_p
    in_elems = n * h * w * cin_p
    out_elems = m_out * cout
    w_elems = cout * r * s * cin_p
    if xe is not None:
        ce = xe.shape[1]
        a.xe, a.we, a.Ce = xe.data_ptr(), we.data_ptr(), ce
        k_total += ce
        in_elems += m_out * ce
        w_elems += cout * ce
    if w2 is not None:
        a.w2, a.y2 = w2.data_ptr(), y2.data_ptr()
        k_total += cin_p
        out_elems += m_out * cout
        w_elems += cout * cin_p
    if residual is not None:
        in_elems += m_out * cout
    if norm is not None:           # (mean [M], rstd [M], wsum [Cout]) fp32: NormConv2d's patch standardisation in the epilogue
        a.norm_mean, a.norm_rstd, a.norm_wsum = norm[0].data_ptr(), norm[1].data_ptr(), norm[2].data_ptr()
    st = st2 = None
    if want_stats:
        st = torch.empty((conv_stat_slots(x.device), cout, 2), device=x.device, dtype=torch.float32)
        a.stats = st.data_ptr()
        if w2 is not None:
            st2 = torch.empty((conv_stat_slots(x.device), cout, 2), device=x.device, dtype=torch.float32)
            a.stats2 = st2.data_ptr()
    slots = ctypes.c_int(0)
    info = dict(shape=(kind, h, cin_p, cout, r, stride), launches=1,
                **conv_work(m_out, cout, k_total, in_elems, w_elems, out_elems))
    check(_timed(kind, info, lambda: lib().hb_conv2d_fused_bf16(ctypes.byref(a), ctypes.byref(slots), stream_ptr())),
          "hb_conv2d_fused_bf16")
    if want_stats:
        if slots.value > st.shape[0]:
            raise RuntimeError("statistics slot capacity exceeded")
        attach_stats(y, st, slots.value)
        if y2 is not None:
            attach_stats(y2, st2, slots.value)
    return y if w2 is None else (y, y2)


class _Conv2dFn(torch.autograd.Function):
    """y = conv2d(x, weight) (+ bias) on the wgmma implicit-GEMM kernels; backward = dgrad + wgrad kernels.

    Channel counts that do not fit the kernels' granularity are zero-padded internally: the input to a multiple of 8
    (or whatever padded width the incoming activation already has), the output to a multiple of 16. With
    ``keep_padded`` the padded output is returned as is (its extra channels are exactly zero), otherwise it is sliced
    back to ``out_channels``. ``want_stats``: the output carries its BatchNorm statistics partials."""

    @staticmethod
    def forward(ctx, x: Tensor, weight: Tensor, bias: Optional[Tensor], stride: int, pad: int, dil: int,
                keep_padded: bool, want_stats: bool = False) -> Tensor:
        cout, cin, r, s = weight.shape
        if x.shape[1] < cin:
            raise RuntimeError(f"expected an input with at least {cin} channels, got {x.shape[1]}")
        need_dx = ctx.needs_input_grad[0]
        if (cin <= 4 and x.shape[1] == cin and r == 3 and s == 3 and pad == 1 and dil == 1 and not need_dx and x.is_contiguous()
                and x.dtype in DTYPE_CODE and cout % 16 == 0 and not os.environ.get("HB_DISABLE_STEM_IM2COL")):
            # network stem (3 input channels): one explicit im2col pass (27 -> 32 columns), then a dense 1x1 GEMM over it. The
            # implicit-GEMM path pads 3 channels to 8-16 and fetches 9 x 32-byte pixels per output through TMA im2col, far below
            # the HBM rate.
            col, wp, _ = _stem_im2col(x, weight, stride)
            y = conv2d_forward_raw(col, wp, cout, 1, 1, 1, 0, 1, _pad_vec(bias, cout),
                                   want_stats=want_stats and epilogue_stats_pay_off(col.shape[1]))
            ctx.save_for_backward(col, weight)
            ctx.cfg = ("stem", bias is not None)
            return y
        y, pk, xb = _packed_conv(x, weight, bias, stride, pad, dil, need_dgrad=need_dx, keep_padded=keep_padded,
                                 want_stats=want_stats)
        ctx.save_for_backward(xb, weight)
        ctx.cfg = (stride, pad, dil, pk.wd, bias is not None, x.shape[1], pk.cout_p, pk.cin_d)
        return y

    @staticmethod
    def backward(ctx, dy: Tensor):
        xb, weight = ctx.saved_tensors
        if ctx.cfg[0] == "stem":
            cout = weight.shape[0]
            dyb = to_channels_last_bf16(dy, cout)
            dw = db = None
            if ctx.needs_input_grad[1]:
                dw = _stem_wgrad(xb, dyb, weight)
            if ctx.cfg[1] and ctx.needs_input_grad[2]:
                db = dyb.float().sum((0, 2, 3))
            return None, dw, db, None, None, None, None, None
        stride, pad, dil, wd, has_bias, cin_x, cout_p, cin_d = ctx.cfg
        cout = weight.shape[0]
        h, w = xb.shape[2], xb.shape[3]
        dyb = to_channels_last_bf16(dy, cout_p)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            if dil != 1:
                raise NotImplementedError("dgrad with dilation > 1")
            dxp = _dgrad(dyb, weight, wd, cin_d, h, w, stride, pad)
            dx = dxp if cin_d == cin_x else dxp[:, :cin_x]
        if ctx.needs_input_grad[1]:
            dw = _wgrad(xb, dyb, weight, stride, pad, dil)
        if has_bias and ctx.needs_input_grad[2]:
            db = dyb[:, :cout].float().sum((0, 2, 3))
        return dx, dw, db, None, None, None, None, None


def conv2d(x: Tensor, weight: Tensor, bias: Optional[Tensor] = None, stride: int = 1, padding: int = 0,
           dilation: int = 1, keep_padded: bool = False, want_stats: bool = False) -> Tensor:
    """Dense (groups=1) 2-D convolution on the sm_90a tensor cores; returns bf16 channels_last."""
    require_cuda(x, weight)
    return _Conv2dFn.apply(x, weight, bias, int(stride), int(padding), int(dilation), bool(keep_padded), bool(want_stats))


def wgrad_raw(xb: Tensor, dyb: Tensor, cout: int, k: int, stride: int, pad: int, dil: int = 1,
              acc_into: Optional[Tensor] = None) -> Optional[Tensor]:
    """fp32 [cout, k, k, cin_p] weight gradient of a conv with NHWC bf16 input ``xb`` and output gradient ``dyb``.

    ``acc_into`` (a KRSC-contiguous fp32 gradient buffer): the reduction kernel ADDS the gradient to it and ``None`` is
    returned; when the shape has no reduction pass to fold the addition into (return code 801) nothing is touched and
    the string ``"unsupported"`` is returned so that the caller computes the gradient separately."""
    n, cin_p, h, w = xb.shape
    L = lib()
    ws_bytes = L.hb_conv2d_wgrad_workspace_bytes(n, h, w, cin_p, cout, k, k, stride, pad, dil, 0)
    ws = torch.empty(ws_bytes // 4, device=xb.device, dtype=torch.float32) if ws_bytes else None
    ho, wo = dyb.shape[2], dyb.shape[3]
    info = dict(shape=("wgrad", h, cin_p, cout, k, stride), launches=1,
                **conv_work(n * ho * wo, cout, k * k * cin_p, n * h * w * cin_p + n * ho * wo * cout, cout * k * k * cin_p,
                            out_elems=0, w_bytes_per=4))
    if acc_into is not None:
        rc = _timed("wgrad", info, lambda: L.hb_conv2d_wgrad_acc_bf16(
            ptr(xb), ptr(dyb), ptr(acc_into), ptr(ws), ws_bytes, n, h, w, cin_p, cout, k, k, stride, pad, dil, 0,
            stream_ptr()))
        if rc == 801:
            return "unsupported"
        check(rc, "hb_conv2d_wgrad_acc_bf16")
        return None
    dwp = torch.empty((cout, k, k, cin_p), device=xb.device, dtype=torch.float32)
    check(_timed("wgrad", info, lambda: L.hb_conv2d_wgrad_bf16(
        ptr(xb), ptr(dyb), ptr(dwp), ptr(ws), ws_bytes, n, h, w, cin_p, cout, k, k, stride, pad, dil, 0, stream_ptr())),
        "hb_conv2d_wgrad_bf16")
    return dwp


def _packed_conv(x: Tensor, weight: Tensor, bias: Optional[Tensor], stride: int, pad: int, dil: int, act: int = ACT_NONE,
                 *, need_dgrad: bool = False, keep_padded: bool = False, want_stats: bool = False, norm=None):
    """Packs ``weight``, converts ``x`` to the packed channel width and runs one convolution -> ``(y, pk, xb)``, ``y``
    sliced to Cout unless ``keep_padded``. ``norm(xb, pk)`` returns the (mean, rstd, wsum) of NormConv2d's epilogue."""
    cout, _, r, s = weight.shape
    pk = pack_filter(weight, need_dgrad, round_up(x.shape[1], 8))
    xb = to_channels_last_bf16(x, pk.cin_p)
    nrm = None if norm is None else norm(xb, pk)
    y = conv2d_forward_raw(xb, pk.wf, pk.cout_p, r, s, stride, pad, dil, _pad_vec(bias, pk.cout_p), None, act,
                           want_stats=want_stats and epilogue_stats_pay_off(r * s * pk.cin_p), norm=nrm)
    return (y if (keep_padded or pk.cout_p == cout) else y[:, :cout]), pk, xb


def _zero_insert(t: Tensor, h: int, w: int, stride: int) -> Tensor:
    """[N, C, h, w] with the pixels of ``t`` at every ``stride``-th position and zeros between them."""
    n, c, ho, wo = t.shape
    out = _empty_cl(n, c, h, w, t.device)
    check(lib().hb_zero_insert_bf16(ptr(t), ptr(out), n, ho, wo, h, w, c, stride, stream_ptr()), "hb_zero_insert_bf16")
    return out


def _dgrad(dyb: Tensor, weight: Tensor, wd: Tensor, cin_d: int, h: int, w: int, stride: int, pad: int,
           dy1: Optional[Tensor] = None, wd1: Optional[Tensor] = None) -> Tensor:
    """dx [N, cin_d, h, w] of a convolution (``weight``, packed for the data gradient as ``wd``) plus that of a RepVGG 1x1
    branch (``dy1``, ``wd1``): parity classes for stride-2 3x3 pad-1 filters, else zero insertion and a convolution with
    the flipped filter (the 1x1 branch convolved at the low resolution, then zero-inserted)."""
    r, s = weight.shape[2], weight.shape[3]
    if stride == 2 and r == 3 and s == 3 and pad == 1 and h >= 2 and w >= 2:
        return dgrad_s2_raw(dyb, weight, cin_d, h, w, dy1, wd1)
    dxa = None
    if dy1 is not None:
        dxa = conv2d_forward_raw(dy1, wd1, cin_d, 1, 1, 1, 0, 1, kind="dgrad")
        if stride > 1:
            dxa = _zero_insert(dxa, h, w, stride)
    src = _zero_insert(dyb, h, w, stride) if stride > 1 else dyb
    dxp = conv2d_forward_raw(src, wd, cin_d, r, s, 1, r - 1 - pad, 1, kind="dgrad")
    if dxa is not None:
        dxp.add_(dxa)
    return dxp


def _wgrad_to_param(dwp: Tensor, weight: Tensor) -> Tensor:
    """KRSC [cout_p, k, k, cin_p] weight gradient -> ``weight``'s (Cout, Cin, k, k), channel padding sliced off."""
    cout, cin = weight.shape[0], weight.shape[1]
    dw = dwp.permute(0, 3, 1, 2)
    if dw.shape[0] != cout or dw.shape[1] != cin:
        dw = dw[:cout, :cin].contiguous(memory_format=torch.channels_last)
    return dw


def _wgrad(xb: Tensor, dyb: Tensor, weight: Tensor, stride: int, pad: int, dil: int = 1) -> Optional[Tensor]:
    """Weight gradient of one filter from the (channel-padded) input and output gradient: ``None`` when the reduction
    kernel added it into the parameter's gradient buffer (:func:`direct_grad`), otherwise in the parameter's shape."""
    cout, cin, r, s = weight.shape
    if r != s:
        raise NotImplementedError("non-square filters")
    cout_p, cin_p = dyb.shape[1], xb.shape[1]
    g = direct_grad(weight, krsc=True) if (cin_p == cin and cout_p == cout) else None
    if g is not None and wgrad_raw(xb, dyb, cout_p, r, stride, pad, dil, acc_into=g) is None:
        return None
    return _wgrad_to_param(wgrad_raw(xb, dyb, cout_p, r, stride, pad, dil), weight)


def conv2d_bias_act(x: Tensor, weight: Tensor, bias: Optional[Tensor], stride: int, padding: int, act: int = ACT_NONE,
                    slope: float = 0.0) -> Tensor:
    """conv + bias + activation. Without autograd (inference) bias and ReLU are fused in the conv epilogue;
    with autograd the activation is applied by the fused pointwise pass."""
    require_cuda(x, weight)
    needs_grad = torch.is_grad_enabled() and (x.requires_grad or weight.requires_grad or
                                              (bias is not None and bias.requires_grad))
    if not needs_grad and act in (ACT_NONE, ACT_RELU):
        return _packed_conv(x, weight, bias, stride, padding, 1, act)[0]
    if act == ACT_NONE:
        return _Conv2dFn.apply(x, weight, bias, int(stride), int(padding), 1, False, False)
    # the activation pass needs channels % 8 == 0: run it on the zero-padded output (filter rows and bias of the padding are
    # zero and every supported activation maps 0 to 0), slice afterwards - identical when Cout % 16 == 0
    y = act_only(_Conv2dFn.apply(x, weight, bias, int(stride), int(padding), 1, True, False), act, slope)
    return y if y.shape[1] == weight.shape[0] else y[:, :weight.shape[0]]


# ------------------------------------------------------------------------------------------------------
BATCH_NORMS = (nn.BatchNorm2d, nn.SyncBatchNorm)


def is_batch_norm(m: nn.Module) -> bool:
    """Whether the fused BatchNorm pass takes ``m``: an ``nn.BatchNorm2d``, or the ``nn.SyncBatchNorm`` that
    ``nn.SyncBatchNorm.convert_sync_batchnorm`` turns it into (not a subclass of it)."""
    return isinstance(m, BATCH_NORMS)


def sync_group(bns: Sequence[nn.Module], training: bool) -> Optional["dist.ProcessGroup"]:
    """The process group whose ranks share the batch statistics of ``bns``, or None for per-GPU statistics.

    ``nn.SyncBatchNorm``'s rule: synchronise only in training (batch statistics), with ``torch.distributed`` initialised
    and more than one rank in the layer's group (``process_group``, default the world). Otherwise a converted layer runs
    the plain BatchNorm path. The branches of one fused pass share one all-reduce, so they must agree on all of this."""
    syncs = [b for b in bns if isinstance(b, nn.SyncBatchNorm)]
    if not training or not syncs or not (dist.is_available() and dist.is_initialized()):
        return None
    group = syncs[0].process_group or dist.group.WORLD
    if dist.get_world_size(group) < 2:
        return None
    if len(syncs) != len(bns) or any(b.process_group is not syncs[0].process_group for b in syncs):
        raise NotImplementedError("one fused BatchNorm pass over branches that do not share one SyncBatchNorm process group")
    return group


def _all_reduce(t: Tensor, group) -> None:
    """SUM all-reduce of ``t`` over ``group``, ordered on the current stream (captured into a CUDA graph like the
    gradient bucket's)."""
    dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)


class BNBranch:
    """Non-tensor view of one BatchNorm2d's buffers/hyper-parameters handed to the fused function."""
    __slots__ = ("running_mean", "running_var", "eps", "momentum", "num_batches_tracked", "track_running_stats")

    def __init__(self, bn: nn.BatchNorm2d) -> None:
        self.running_mean = bn.running_mean
        self.running_var = bn.running_var
        self.eps = bn.eps
        self.momentum = bn.momentum
        self.num_batches_tracked = bn.num_batches_tracked
        # nn.BatchNorm2d updates its buffers in training only while the flag is set (trainer.freeze_bn clears it)
        self.track_running_stats = bn.track_running_stats and bn.running_mean is not None


def _arr3(ts: Sequence[Optional[Tensor]]):
    vals = [0 if t is None else t.data_ptr() for t in ts]
    return _VP3(*(vals + [0] * (3 - len(vals))))


_I3 = ctypes.c_int * 3


def _elem_bytes_info(kind: str, m: int, c: int, reads: int, writes: int) -> dict:
    """Algorithmic HBM bytes of a streaming pass over [m, c] bf16 tensors: ``reads`` tensors in, ``writes`` out."""
    return dict(shape=(kind, m, c, reads, writes), launches=1, flops=0.0, bytes=2.0 * m * c * (reads + writes))


def _bn_batch_stats(us: Sequence[Tensor], branches, g32, b32, stats: Tensor, c: int, c_log: int, m: int,
                    group=None) -> Optional[Tensor]:
    """Training-mode statistics -> mean / rstd / scale / shift rows of ``stats`` (+ running-statistics update).

    Every input normally arrives with its (sum, sum of squares) partials attached by its producer (convolution epilogue,
    previous block's forward pass); only tensors that come without them get a stand-alone statistics pass.

    ``group`` (:func:`sync_group`): the branches' fp64 sums and row count are packed into one buffer, all-reduced over
    the group (one collective for every branch) and finalised from the global values; the buffer is returned (its last
    element, the global row count, is what the backward pass normalises by). Without a group: None."""
    if m == 1 and group is None:   # what F.batch_norm raises in training: the variance of one value is undefined
        raise ValueError(f"Expected more than 1 value per channel when training, got input size {us[0].shape}")
    L = lib()
    nb = len(us)
    parts, slots = [], []
    for u in us:
        st = get_stats(u)
        if st is None:
            buf = torch.empty((bn_stat_slots(u.device), c, 2), device=u.device, dtype=torch.float32)
            sl = ctypes.c_int(0)
            check(_timed("bn_stats", _elem_bytes_info("bn_stats", m, c, 1, 0), lambda: L.hb_bn_stats_partials_bf16(
                ptr(u), m, c, ptr(buf), ctypes.byref(sl), stream_ptr())), "hb_bn_stats_partials_bf16")
            st = (buf, sl.value)
        parts.append(st[0])
        slots.append(st[1])
    eps, mom = branches[0].eps, branches[0].momentum
    if any(b.eps != eps or b.momentum != mom for b in branches):
        raise NotImplementedError("branches with different eps/momentum")
    track = [b.track_running_stats for b in branches]
    if mom is None and any(track):
        raise NotImplementedError("cumulative moving average (momentum=None)")
    running = (_arr3([b.running_mean if t else None for b, t in zip(branches, track)]),
               _arr3([b.running_var if t else None for b, t in zip(branches, track)]),
               _arr3([b.num_batches_tracked if t else None for b, t in zip(branches, track)]))
    outs = (ptr(stats[0]), ptr(stats[1]), ptr(stats[2]), ptr(stats[3]))
    if group is None:
        check(L.hb_bn_finalize(_arr3(parts), _I3(*(slots + [0] * (3 - nb))), _arr3(g32), _arr3(b32), *running, *outs, nb, c,
                               c_log, m, _c_float(eps), _c_float(0.0 if mom is None else mom), stream_ptr()),
              "hb_bn_finalize")
        return None
    sums = sync_sums_buffer(nb, c, stats.device)
    check(L.hb_bn_partials_sums(_arr3(parts), _I3(*(slots + [0] * (3 - nb))), nb, c, c_log, m, ptr(sums), stream_ptr()),
          "hb_bn_partials_sums")
    _all_reduce(sums, group)
    check(L.hb_bn_finalize_sums(ptr(sums), _arr3(g32), _arr3(b32), *running, *outs, nb, c, c_log, _c_float(eps),
                                _c_float(0.0 if mom is None else mom), stream_ptr()), "hb_bn_finalize_sums")
    return sums


def sync_sums_buffer(nb: int, c: int, device) -> Tensor:
    """fp64 buffer of one synchronised statistics all-reduce: [nb][c][2] (sum, sum of squares), then the row count."""
    return torch.empty(nb * c * 2 + 1, device=device, dtype=torch.float64)


def sync_count(sums: Tensor) -> Tensor:
    """The row count element of a :func:`sync_sums_buffer` (after the all-reduce: the rows of every rank)."""
    return sums[-1:]


def sync_grad_sums(scratch: Tensor, nb: int, c: int) -> Tensor:
    """The [1 + nb][c] (sum dz, sum dz*u_b) head of the backward scratch: what a synchronised backward all-reduces (the
    per-block partials behind it stay local)."""
    return scratch[:(1 + nb) * c]


def _bn_forward_pass(us: Sequence[Tensor], stats: Tensor, res: Optional[Tensor], m: int, c: int, act: int, slope: float,
                     res_after: int, shape, emit_stats: bool) -> Tensor:
    n, _, h, w = shape
    nb = len(us)
    dev = us[0].device if nb else res.device
    if emit_stats and os.environ.get("HB_DISABLE_BN_OUT_STATS"):    # A/B switch
        emit_stats = False
    out = _empty_cl(n, c, h, w, dev)
    ost = torch.empty((bn_stat_slots(dev), c, 2), device=dev, dtype=torch.float32) if emit_stats else None
    sl = ctypes.c_int(0)
    up = [ptr(us[i]) if i < nb else ptr(None) for i in range(3)]
    check(_timed("bn_fwd", _elem_bytes_info("bn_fwd", m, c, nb + (res is not None), 1), lambda: lib().hb_bn_act_fwd_bf16(
        up[0], up[1], up[2], nb, ptr(stats[2]), ptr(stats[3]), ptr(res), ptr(out), m, c, act, _c_float(slope), int(res_after),
        ptr(ost), ctypes.byref(sl) if emit_stats else None, stream_ptr())), "hb_bn_act_fwd_bf16")
    if emit_stats:
        attach_stats(out, ost, sl.value)
    return out


def _bn_backward_pass(dob: Tensor, us: Sequence[Tensor], stats: Tensor, res: Optional[Tensor], dus, dres, dgb, gacc, bacc,
                      c_log: int, m: int, c: int, act: int, slope: float, training: bool, res_after: int,
                      sync=None) -> None:
    """Two streaming passes (reduce, apply) + the C-sized finalisation between them (fixed-order, no atomics).

    ``sync`` = (group, forward sums buffer) of a synchronised BatchNorm: the reduce pass' (sum dz, sum dz*u_b) are
    all-reduced over the group before the apply pass, which normalises by the global row count. The BatchNorm parameter
    gradients stay the local sums, as with ``nn.SyncBatchNorm``: the gradient all-reduce averages them over the ranks."""
    if sync is not None:
        _bn_backward_sync(dob, us, stats, res, dus, dres, dgb, gacc, bacc, c_log, m, c, act, slope, res_after, *sync)
        return
    L = lib()
    nb = len(us)
    scratch = torch.empty(L.hb_bn_bwd_scratch_doubles(m, c, nb), device=dob.device, dtype=torch.float64)
    up = [ptr(us[i]) if i < nb else ptr(None) for i in range(3)]
    dup = [ptr(dus[i]) if i < nb else ptr(None) for i in range(3)]
    nres = int(res is not None and not res_after)
    nwr = sum(d is not None for d in dus) + (dres is not None)
    # reduce pass reads dout + inputs (+ residual inside the activation); apply pass reads them again and writes gradients
    info = _elem_bytes_info("bn_bwd", m, c, 2 * (1 + nb + nres), nwr)
    info["launches"] = 3
    check(_timed("bn_bwd", info, lambda: L.hb_bn_act_bwd_bf16(
        ptr(dob), up[0], up[1], up[2], nb, ptr(stats[2]), ptr(stats[3]), ptr(stats[0]), ptr(stats[1]), ptr(res), ptr(scratch),
        dup[0], dup[1], dup[2], ptr(dres), ptr(dgb[0]) if dgb is not None else ptr(None),
        ptr(dgb[1]) if dgb is not None else ptr(None), _arr3(gacc) if gacc is not None else None,
        _arr3(bacc) if bacc is not None else None, c_log, m, c, act, _c_float(slope), 1 if training else 0, res_after,
        stream_ptr())), "hb_bn_act_bwd_bf16")


def _bn_backward_sync(dob: Tensor, us: Sequence[Tensor], stats: Tensor, res: Optional[Tensor], dus, dres, dgb, gacc, bacc,
                      c_log: int, m: int, c: int, act: int, slope: float, res_after: int, group, fwd_sums: Tensor) -> None:
    L = lib()
    nb = len(us)
    scratch = torch.empty(L.hb_bn_bwd_scratch_doubles(m, c, nb), device=dob.device, dtype=torch.float64)
    up = [ptr(us[i]) if i < nb else ptr(None) for i in range(3)]
    dup = [ptr(dus[i]) if i < nb else ptr(None) for i in range(3)]
    nres = int(res is not None and not res_after)
    nwr = sum(d is not None for d in dus) + (dres is not None)
    info = _elem_bytes_info("bn_bwd", m, c, 1 + nb + nres, 0)
    info["launches"] = 2
    check(_timed("bn_bwd", info, lambda: L.hb_bn_act_bwd_reduce_bf16(
        ptr(dob), up[0], up[1], up[2], nb, ptr(stats[2]), ptr(stats[3]), ptr(stats[0]), ptr(stats[1]), ptr(res), ptr(scratch),
        ptr(dgb[0]) if dgb is not None else ptr(None), ptr(dgb[1]) if dgb is not None else ptr(None),
        _arr3(gacc) if gacc is not None else None, _arr3(bacc) if bacc is not None else None, c_log, m, c, act,
        _c_float(slope), res_after, stream_ptr())), "hb_bn_act_bwd_reduce_bf16")
    _all_reduce(sync_grad_sums(scratch, nb, c), group)
    info = _elem_bytes_info("bn_bwd", m, c, 1 + nb + nres, nwr)
    check(_timed("bn_bwd", info, lambda: L.hb_bn_act_bwd_apply_bf16(
        ptr(dob), up[0], up[1], up[2], nb, ptr(stats[2]), ptr(stats[3]), ptr(stats[0]), ptr(stats[1]), ptr(res), ptr(scratch),
        ptr(sync_count(fwd_sums)), dup[0], dup[1], dup[2], ptr(dres), m, c, act, _c_float(slope), res_after, stream_ptr())),
        "hb_bn_act_bwd_apply_bf16")


def _bn_setup(us: Sequence[Tensor], branches, gammas: Sequence[Tensor], betas: Sequence[Tensor], training: bool, c: int,
              c_log: int, m: int, dev, group=None) -> Tuple[Tensor, Optional[Tensor]]:
    """[4, max(nb, 1), c] fp32 mean / rstd / scale / shift rows of the branches: batch statistics in training, the
    running statistics otherwise. ``c_log``: the parameters' channel count (<= c, the activation's padded width).
    Returns them with the all-reduced sums of a synchronised BatchNorm (``group``, :func:`_bn_batch_stats`) or None."""
    stats = torch.empty((4, max(len(branches), 1), c), device=dev, dtype=torch.float32)
    g32 = [g.detach().float() for g in gammas]
    b32 = [b.detach().float() for b in betas]
    if not branches:
        return stats, None
    if training:
        return stats, _bn_batch_stats(us, branches, g32, b32, stats, c, c_log, m, group)
    for i, b in enumerate(branches):
        check(lib().hb_bn_eval_affine(ptr(g32[i]), ptr(b32[i]), ptr(b.running_mean), ptr(b.running_var), _c_float(b.eps), c,
                                      c_log, ptr(stats[2][i]), ptr(stats[3][i]), ptr(stats[0][i]), ptr(stats[1][i]),
                                      stream_ptr()), "hb_bn_eval_affine")
    return stats, None


def _bn_grad_targets(gammas: Sequence[Tensor], betas: Sequence[Tensor], c: int, dev):
    """(gacc, bacc, dgb) of the BatchNorm weights / biases: their gradient buffers when the kernel may add into all of
    them (``dgb`` None), otherwise a [2, nb, c] fp32 buffer the kernel writes the gradients to (``gacc``, ``bacc`` None)."""
    gacc = [direct_grad(p) for p in gammas]
    bacc = [direct_grad(p) for p in betas]
    if all(g is not None for g in gacc) and all(b is not None for b in bacc):
        return gacc, bacc, None
    return None, None, torch.empty((2, len(gammas), c), device=dev, dtype=torch.float32)


class _BNActFn(torch.autograd.Function):
    """out = act(sum_b BN_b(u_b) [+ residual]); training (batch statistics) or eval (running statistics)."""

    @staticmethod
    def forward(ctx, cfg, *tensors: Tensor) -> Tensor:
        branches, act, slope, training, has_res, res_after, emit_stats, group = cfg
        nb = len(branches)
        us = [to_channels_last_bf16(t) for t in tensors[:nb]]
        gammas = tensors[nb:2 * nb]
        betas = tensors[2 * nb:3 * nb]
        res = to_channels_last_bf16(tensors[3 * nb]) if has_res else None
        n, c, h, w = us[0].shape if nb else res.shape
        if c % 8 != 0:
            raise NotImplementedError("fused BN kernels need channels % 8 == 0")
        m = n * h * w
        dev = us[0].device if nb else res.device
        c_log = gammas[0].numel() if nb else c   # parameters may be narrower than a zero-padded activation
        stats, sums = _bn_setup(us, branches, gammas, betas, training, c, c_log, m, dev, group)
        out = _bn_forward_pass(us, stats, res, m, c, act, slope, int(res_after), (n, c, h, w), emit_stats)
        ctx.save_for_backward(stats, *us, *([res] if has_res else []), *gammas, *betas)
        ctx.cfg = (nb, act, slope, training, has_res, c_log, int(res_after))
        ctx.sync = None if sums is None else (group, sums)
        return out

    @staticmethod
    def backward(ctx, dout: Tensor):
        nb, act, slope, training, has_res, c_log, res_after = ctx.cfg
        saved = ctx.saved_tensors
        stats, us = saved[0], saved[1:1 + nb]
        res = saved[1 + nb] if has_res else None
        params = saved[1 + nb + int(has_res):]
        gammas, betas = params[:nb], params[nb:]
        n, c, h, w = us[0].shape if nb else res.shape
        m = n * h * w
        dev = dout.device
        dob = to_channels_last_bf16(dout)
        need_u = [ctx.needs_input_grad[1 + i] for i in range(nb)]
        need_gb = any(ctx.needs_input_grad[1 + nb:1 + 3 * nb])
        need_res = has_res and ctx.needs_input_grad[1 + 3 * nb]
        dus = [_empty_cl(n, c, h, w, dev) if need_u[i] else None for i in range(nb)]
        dres = _empty_cl(n, c, h, w, dev) if need_res else None
        gacc, bacc, dgb = _bn_grad_targets(gammas, betas, c, dev) if need_gb else (None, None, None)
        _bn_backward_pass(dob, us, stats, res, dus, dres, dgb, gacc, bacc, c_log, m, c, act, slope, training, res_after,
                          ctx.sync)
        grads: List[Optional[Tensor]] = [None]
        grads += dus
        grads += [dgb[0][i][:c_log] if dgb is not None else None for i in range(nb)]
        grads += [dgb[1][i][:c_log] if dgb is not None else None for i in range(nb)]
        if has_res:
            grads.append(dres)
        return tuple(grads)


def bn_act(us: Sequence[Tensor], bns: Sequence[nn.BatchNorm2d], act: int = ACT_NONE, slope: float = 0.0,
           residual: Optional[Tensor] = None, training: Optional[bool] = None, res_after_act: bool = False,
           emit_stats: bool = False) -> Tensor:
    """act(sum_b BatchNorm_b(u_b) + residual) as one fused pass (training: the statistics come with the inputs from the
    kernels that produced them, see :func:`get_stats`); ``res_after_act`` moves the residual outside the activation:
    act(sum_b ...) + residual. ``emit_stats``: the output carries its own statistics partials. ``bns`` may be
    ``nn.SyncBatchNorm`` layers: their statistics are then shared over their process group (:func:`sync_group`)."""
    if not 1 <= len(us) <= 3 or len(us) != len(bns):
        raise ValueError("between 1 and 3 (input, BatchNorm2d) pairs are supported")
    require_cuda(*us)
    if training is None:
        training = bns[0].training
    use_batch_stats = training or bns[0].running_mean is None
    cfg = ([BNBranch(b) for b in bns], int(act), float(slope), bool(use_batch_stats), residual is not None,
           bool(res_after_act), bool(emit_stats), sync_group(bns, training))
    args = list(us) + [b.weight for b in bns] + [b.bias for b in bns]
    if residual is not None:
        args.append(residual)
    return _BNActFn.apply(cfg, *args)


def act_only(x: Tensor, act: int, slope: float = 0.0) -> Tensor:
    """Stand-alone activation through the fused pass (zero BN branches, x as the residual input)."""
    cfg = ([], int(act), float(slope), False, True, False, False, None)
    return _BNActFn.apply(cfg, x)


# ------------------------------------------------------------------------------------------------------
class _RepBlockFn(torch.autograd.Function):
    """Train-form RepVGG block as ONE autograd node:  out = act(BN3(conv3x3(x)) + BN1(conv1x1(x)) [+ BNid(x)]).

    Forward: ONE tensor-core launch computes both branches from a single read of x (the 1x1 branch re-uses the centre-tap
    loads of the 3x3 branch into a second accumulator) and its epilogue also produces the BatchNorm statistics of both
    outputs; the identity branch's statistics arrive with x from the previous block's forward pass. Then one C-sized
    finalisation and ONE fused pass that normalises the branches, sums them, applies the activation and accumulates the
    statistics of its own output for the next block (reference: 2 cuDNN convs + 3 BatchNorm kernels + 2 adds + ReLU).

    Backward: instead of letting autograd sum the three input-gradient contributions with two extra element-wise
    kernels, they are produced by one launch
        dX = dgrad3x3(dY3) + dgrad1x1(dY1)  [K extension]  + dXid  [epilogue residual]
    (stride-2 blocks: parity-class data gradient with the 1x1 branch accumulated into class (0, 0)); both weight
    gradients come from one pass over x and are added straight into the parameters' gradient buffers when those are
    bound to a :class:`holocron_b200.distributed.GradBucket`.
    """

    @staticmethod
    def forward(ctx, cfg, x: Tensor, w3: Tensor, w1: Tensor, *bn_params: Tensor) -> Tensor:
        branches, act, slope, training, stride, group = cfg
        nb = len(branches)
        gammas, betas = bn_params[:nb], bn_params[nb:]
        need_dx = ctx.needs_input_grad[1]
        cout, cin = w3.shape[0], w3.shape[1]
        if cout % 16 != 0:
            raise NotImplementedError("fused RepBlock needs out_channels % 16 == 0")
        stem = cin <= 4 and x.shape[1] == cin and not need_dx and x.is_contiguous() and x.dtype in DTYPE_CODE
        if stem:
            # network stem: explicit im2col once (27 -> 32 columns), both branches become dense 1x1 GEMMs over it
            xb, wf3, wf1 = _stem_im2col(x, w3, stride, w1)
            k3, conv_stride, pad3 = 1, 1, 0
            wd3 = wd1 = None
        else:
            pk3 = pack_filter(w3, need_dx, round_up(x.shape[1], 8))
            pk1 = pack_filter(w1, need_dx, round_up(x.shape[1], 8))
            xb = to_channels_last_bf16(x, pk3.cin_p)
            wf3, wf1, wd3, wd1 = pk3.wf, pk1.wf, pk3.wd, pk1.wd
            k3, conv_stride, pad3 = 3, stride, 1
        kx = xb.shape[1]
        # Dual-output launch (x read once, 1x1 branch from the centre-tap loads): correct and tested, opt-in (A/B). The two
        # accumulators share the 128-column register budget, so each output's Cout tile is capped at 64 columns (twice the
        # tiles on the wide layers) and every tile runs two epilogues; two launches are the default. Not measured on the H100.
        if os.environ.get("HB_FUSED_FPROP"):
            y3, y1 = conv2d_forward_raw(xb, wf3, cout, k3, k3, conv_stride, pad3, 1, w2=wf1,
                                        want_stats=training and epilogue_stats_pay_off(k3 * k3 * kx))
        else:
            y3 = conv2d_forward_raw(xb, wf3, cout, k3, k3, conv_stride, pad3, 1,
                                    want_stats=training and epilogue_stats_pay_off(k3 * k3 * kx))
            y1 = conv2d_forward_raw(xb, wf1, cout, 1, 1, conv_stride, 0, 1,
                                    want_stats=training and epilogue_stats_pay_off(kx))
        us = [y3, y1] + ([xb] if nb == 3 else [])
        n, c, h, w = y3.shape
        m = n * h * w
        stats, sums = _bn_setup(us, branches, gammas, betas, training, c, c, m, y3.device, group)
        out = _bn_forward_pass(us, stats, None, m, c, act, slope, 0, (n, c, h, w), emit_stats=training)
        ctx.save_for_backward(stats, xb, y3, y1, w3, w1, *gammas, *betas)
        ctx.cfg = (nb, act, slope, training, stride, wd3, wd1, x.shape[1], stem)
        ctx.sync = None if sums is None else (group, sums)
        return out

    @staticmethod
    def backward(ctx, dout: Tensor):
        nb, act, slope, training, stride, wd3, wd1, cin_x, stem = ctx.cfg
        stats, xb, y3, y1, w3, w1 = ctx.saved_tensors[:6]
        gammas, betas = ctx.saved_tensors[6:6 + nb], ctx.saved_tensors[6 + nb:6 + 2 * nb]
        n, c, ho, wo = y3.shape
        _, cin_p, h, w = xb.shape
        m = n * ho * wo
        dev = dout.device
        L = lib()
        dob = to_channels_last_bf16(dout)
        need_dx = ctx.needs_input_grad[1]
        dy3, dy1 = _empty_cl(n, c, ho, wo, dev), _empty_cl(n, c, ho, wo, dev)
        dxid = _empty_cl(n, c, ho, wo, dev) if (nb == 3 and need_dx) else None
        gacc, bacc, dgb = _bn_grad_targets(gammas, betas, c, dev)
        us = [y3, y1] + ([xb] if nb == 3 else [])
        _bn_backward_pass(dob, us, stats, None, [dy3, dy1] + ([dxid] if nb == 3 else []), None, dgb, gacc, bacc, c, m, c, act,
                          slope, training, 0, ctx.sync)
        g_gamma = [None if dgb is None else dgb[0][i] for i in range(nb)]
        g_beta = [None if dgb is None else dgb[1][i] for i in range(nb)]
        dx = None
        if need_dx:
            cin_d = wd3.shape[0]
            if stride == 1 and wd3.shape[3] == c and (dxid is None or cin_d == c):
                dxp = None
                if not os.environ.get("HB_DISABLE_CONV_ROWS"):
                    # shared-memory-resident filter variant (C <= 64): all three contributions in the K loop
                    eye = _identity_filter(cin_d, c, dev) if dxid is not None else None
                    dxr = _empty_cl(n, cin_d, h, w, dev)
                    nsrc = 2 if dxid is not None else 1
                    info = dict(shape=("dgrad_rows", h, c, cin_d, 3, 1), launches=1,
                                **conv_work(n * h * w, cin_d, 10 * c, (1 + nsrc) * n * h * w * c, 10 * cin_d * c))
                    rc = _timed("dgrad", info, lambda: L.hb_conv3x3_accum_bf16(
                        ptr(dy3), ptr(wd3), ptr(dy1), ptr(wd1), ptr(dxid), ptr(eye), nsrc, ptr(dxr), n, h, w, c, cin_d, 0,
                        stream_ptr()))
                    if rc == 0:
                        dxp = dxr
                    elif rc != 801:   # 801 = cudaErrorNotSupported: shape not eligible for the resident-filter scheme
                        check(rc, "hb_conv3x3_accum_bf16")
                if dxp is None:
                    # generic kernel, one launch: K loop = 9 taps of dY3 + the 1x1 branch's dY1, identity gradient added
                    # in the epilogue
                    dxp = conv2d_forward_raw(dy3, wd3, cin_d, 3, 3, 1, 1, 1, None, dxid, ACT_NONE, xe=dy1, we=wd1, kind="dgrad")
            else:
                # stride 2: parity classes, the 1x1 branch landing in class (0, 0); otherwise (channel-padded or odd
                # shapes) the general composition
                dxp = _dgrad(dy3, w3, wd3, cin_d, h, w, stride, 1, dy1, wd1)
                if dxid is not None:
                    dxp[:, :c].add_(dxid)
            dx = dxp if cin_d == cin_x else dxp[:, :cin_x]
        if stem:
            return (None, None, _stem_wgrad(xb, dy3, w3), _stem_wgrad(xb, dy1, w1), *g_gamma, *g_beta)
        grads_w: List[Optional[Tensor]] = [None, None]
        done = [False, False]
        no_pad = cin_p == w3.shape[1]
        gw3 = direct_grad(w3, krsc=True) if no_pad else None
        gw1 = direct_grad(w1, krsc=True) if no_pad else None
        if stride == 1 and not os.environ.get("HB_DISABLE_FUSED_WGRAD"):
            # both branches' weight gradients in one pass over x (the 1x1 branch = centre-tap window of the same rows)
            ws_bytes = L.hb_repvgg_wgrad_workspace_bytes(n, h, w, cin_p, c, 0)
            if ws_bytes:
                ws = torch.empty(ws_bytes // 4, device=dev, dtype=torch.float32)
                info = dict(shape=("wgrad_rows", h, cin_p, c, 3, 1), launches=2,
                            **conv_work(n * h * w, c, 10 * cin_p, n * h * w * (cin_p + 2 * c), 10 * c * cin_p, out_elems=0,
                                        w_bytes_per=4))
                if gw3 is not None and gw1 is not None:
                    rc = _timed("wgrad", info, lambda: L.hb_repvgg_wgrad_acc_bf16(
                        ptr(xb), ptr(dy3), ptr(dy1), ptr(gw3), ptr(gw1), ptr(ws), ws_bytes, n, h, w, cin_p, c, 0, stream_ptr()))
                    if rc == 0:
                        done = [True, True]
                    elif rc != 801:
                        check(rc, "hb_repvgg_wgrad_acc_bf16")
                else:
                    dwcat = torch.empty(c * 10 * cin_p, device=dev, dtype=torch.float32)
                    rc = _timed("wgrad", info, lambda: L.hb_repvgg_wgrad_bf16(
                        ptr(xb), ptr(dy3), ptr(dy1), ptr(dwcat), ptr(ws), ws_bytes, n, h, w, cin_p, c, 0, stream_ptr()))
                    if rc == 0:
                        grads_w = [_wgrad_to_param(dwcat[:c * 9 * cin_p].view(c, 3, 3, cin_p), w3),
                                   _wgrad_to_param(dwcat[c * 9 * cin_p:].view(c, 1, 1, cin_p), w1)]
                        done = [True, True]
                    elif rc != 801:
                        check(rc, "hb_repvgg_wgrad_bf16")
        for i, (wt, dy, pad) in enumerate(((w3, dy3, 1), (w1, dy1, 0))):
            if not done[i]:
                grads_w[i] = _wgrad(xb, dy, wt, stride, pad)
        return (None, dx, grads_w[0], grads_w[1], *g_gamma, *g_beta)


_eye_cache = {}


def _identity_filter(rows: int, cols: int, device) -> Tensor:
    """[rows, 1, 1, cols] bf16 filter that is the identity on the first min(rows, cols) channels."""
    key = (rows, cols, str(device))
    if key not in _eye_cache:
        _eye_cache[key] = torch.eye(rows, cols, device=device, dtype=torch.bfloat16).reshape(rows, 1, 1, cols).contiguous()
    return _eye_cache[key]


def _stem_im2col(x: Tensor, w3: Tensor, stride: int, w1: Optional[Tensor] = None):
    """x (N, C<=4, H, W) NCHW -> im2col matrix of a 3x3 / pad-1 convolution as a channels_last (N, 32, Ho, Wo) bf16
    tensor, plus the filter and, for a RepVGG block, its 1x1 branch ``w1`` re-expressed as [Cout, 1, 1, 32] rows over its
    columns (k = (r*3 + s)*C + c; the 1x1 branch only touches the centre tap). Returns (col, w3p, w1p or None)."""
    n, cin, h, w = x.shape
    cout = w3.shape[0]
    kp = round_up(9 * cin, 32)
    ho, wo = conv_out_size(h, 3, stride, 1, 1), conv_out_size(w, 3, stride, 1, 1)
    col = _empty_cl(n, kp, ho, wo, x.device)
    check(lib().hb_im2col_smallc_bf16(ptr(x), ptr(col), n, cin, h, w, 3, 3, stride, 1, kp, dtype_code(x), stream_ptr()),
          "hb_im2col_smallc_bf16")
    w3p = torch.zeros((cout, 1, 1, kp), device=x.device, dtype=torch.bfloat16)
    w3p.view(cout, kp)[:, :9 * cin] = w3.detach().permute(0, 2, 3, 1).reshape(cout, 9 * cin)
    w1p = None
    if w1 is not None:
        w1p = torch.zeros((cout, 1, 1, kp), device=x.device, dtype=torch.bfloat16)
        w1p.view(cout, kp)[:, 4 * cin:5 * cin] = w1.detach().reshape(cout, cin)
    return col, w3p, w1p


def _stem_wgrad(col: Tensor, dyb: Tensor, weight: Tensor) -> Tensor:
    """Gradient of a stem filter (3x3, or a RepVGG 1x1 branch at the centre tap) from the im2col columns it was applied
    to: one 1x1 weight gradient over the columns, sliced back to the filter."""
    cout, cin, k = weight.shape[0], weight.shape[1], weight.shape[2]
    g = wgrad_raw(col, dyb, cout, 1, 1, 0).view(cout, -1)
    if k == 1:
        return g[:, 4 * cin:5 * cin].reshape(cout, cin, 1, 1)
    return g[:, :9 * cin].view(cout, 3, 3, cin).permute(0, 3, 1, 2)


def repblock(x: Tensor, w3: Tensor, w1: Tensor, bns: Sequence[nn.BatchNorm2d], stride: int, act: int, slope: float,
             training: bool) -> Tensor:
    """Fused train-form RepVGG block (see :class:`_RepBlockFn`). ``bns`` = [bn3, bn1] or [bn3, bn1, bn_identity], all
    ``nn.BatchNorm2d`` or all ``nn.SyncBatchNorm`` (one statistics all-reduce for the three branches)."""
    require_cuda(x, w3, w1)
    use_batch_stats = training or bns[0].running_mean is None
    cfg = ([BNBranch(b) for b in bns], int(act), float(slope), bool(use_batch_stats), int(stride), sync_group(bns, training))
    return _RepBlockFn.apply(cfg, x, w3, w1, *[b.weight for b in bns], *[b.bias for b in bns])


# ------------------------------------------------------------------------------------------------------
class _GapFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor) -> Tensor:
        xb = to_channels_last_bf16(x)
        n, c, h, w = xb.shape
        y = torch.empty((n, c), device=xb.device, dtype=torch.bfloat16)
        check(lib().hb_gap_fwd_bf16(ptr(xb), ptr(y), n, h * w, c, stream_ptr()), "hb_gap_fwd_bf16")
        ctx.shape = (n, c, h, w)
        return y

    @staticmethod
    def backward(ctx, dy: Tensor):
        n, c, h, w = ctx.shape
        dyb = dy.to(torch.bfloat16).contiguous()
        dx = _empty_cl(n, c, h, w, dy.device)
        check(lib().hb_gap_bwd_bf16(ptr(dyb), ptr(dx), n, h * w, c, stream_ptr()), "hb_gap_bwd_bf16")
        return dx


class _GateActFn(torch.autograd.Function):
    """out = act(x * gate) with gate broadcast over space (squeeze-excite), one pass forward, one pass backward."""

    @staticmethod
    def forward(ctx, x: Tensor, gate: Tensor, act: int, slope: float) -> Tensor:
        xb = to_channels_last_bf16(x)
        n, c, h, w = xb.shape
        g = gate.detach().reshape(n, c).float().contiguous()
        out = _empty_cl(n, c, h, w, xb.device)
        check(lib().hb_gate_act_fwd_bf16(ptr(xb), ptr(g), ptr(out), n, h * w, c, act, _c_float(slope), stream_ptr()),
              "hb_gate_act_fwd_bf16")
        ctx.save_for_backward(xb, g)
        ctx.cfg = (act, slope, gate.dtype, tuple(gate.shape))
        return out

    @staticmethod
    def backward(ctx, dout: Tensor):
        xb, g = ctx.saved_tensors
        act, slope, gdtype, gshape = ctx.cfg
        n, c, h, w = xb.shape
        dob = to_channels_last_bf16(dout)
        dx = _empty_cl(n, c, h, w, xb.device)
        dg = torch.empty((n, c), device=xb.device, dtype=torch.float32)
        check(lib().hb_gate_act_bwd_bf16(ptr(dob), ptr(xb), ptr(g), ptr(dx), ptr(dg), n, h * w, c, act, _c_float(slope),
                                         stream_ptr()), "hb_gate_act_bwd_bf16")
        return dx, dg.to(gdtype).reshape(gshape), None, None


def gate_act(x: Tensor, gate: Tensor, act: int = ACT_NONE, slope: float = 0.0) -> Tensor:
    """act(x * gate): x (N, C, H, W), gate (N, C, 1, 1) — SEBlock's `x * y` fused with the activation that follows it
    (reference rexnet.py:63-66 + 125-131)."""
    require_cuda(x, gate)
    if gate.shape[:2] != x.shape[:2] or gate.numel() != x.shape[0] * x.shape[1]:
        raise ValueError(f"gate of shape {tuple(gate.shape)} does not match input {tuple(x.shape)}")
    return _GateActFn.apply(x, gate, int(act), float(slope))


def head_linear(feats: Tensor, weight: Tensor, bias: Optional[Tensor]) -> Tensor:
    """Classifier head: plain library GEMM in the activation dtype (bf16 operands, fp32 accumulation, bf16 result), logits
    returned in fp32 (the head ``Linear`` of RepVGG / ReXNet / Darknet; not a hot-path kernel, see DESIGN.md)."""
    import torch.nn.functional as TF
    return TF.linear(feats, weight.to(feats.dtype), None if bias is None else bias.to(feats.dtype)).float()


def global_avg_pool_flat(x: Tensor) -> Tensor:
    """(N, C, H, W) -> (N, C) mean over space (bf16 channels_last in, bf16 out; fp32 accumulation)."""
    return _GapFn.apply(x)
