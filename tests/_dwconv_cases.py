"""The depth-wise convolution cases and a Python mirror of the dispatch and grid geometry of csrc/dwconv.cu (no GPU).

``route`` names the kernel each direction of a case takes and the grid it gets, the way ``narrow_n_tiles`` /
``fprop_slots`` mirror conv_fprop.cu: the launcher conditions of ``hb_dwconv_fwd_bf16``, ``hb_dwconv_bwd_data_bf16``
and ``hb_dwconv_bwd_weight_bf16``, their ``SlabGeo::grid`` arguments (the slab geometry itself is mirrored in
tests/_slab.py) and ``stream_grid``. Every kernel is grid-stride: a thread starting at item ``i0 < S`` (S = grid x items per block) runs
``ceil((total - i0) / S)`` iterations, at least ``total // S`` and at most ``ceil(total / S)``. The SM count sizes the
grids, so the mirror takes it as an argument (H100 SXM: 132, H100 PCIe: 114)."""
from dataclasses import dataclass
from typing import Dict, List, Optional

import _slab as S

THREADS = 256
INT_MAX = 0x7FFFFFFF

# every kernel instantiation in dwconv.cu, and dw_weight_finalize_kernel's four-way unrolled loop counted separately
INSTANTIATIONS = (
    "dw_fwd_kernel",
    "dw_bwd_data_kernel",
    "dw3x3_kernel<false,1>", "dw3x3_kernel<false,2>", "dw3x3_kernel<false,0>",
    "dw3x3_kernel<true,1>", "dw3x3_kernel<true,2>", "dw3x3_kernel<true,0>",
    "dw3x3_quad_kernel<1,false>", "dw3x3_quad_kernel<2,false>", "dw3x3_quad_kernel<1,true>",
    "dw3x3_dgrad_s2_quad_kernel",
    "dw_bwd_weight_kernel<1>", "dw_bwd_weight_kernel<3>", "dw_bwd_weight_kernel<5>", "dw_bwd_weight_kernel<7>",
    "dw3x3_wgrad_quad_kernel<1>", "dw3x3_wgrad_quad_kernel<2>",
    "dw_weight_finalize_kernel",
)
FINALIZE_UNROLLED = "dw_weight_finalize_kernel/unrolled"


@dataclass(frozen=True)
class Case:
    n: int
    c: int
    h: int
    w: int
    k: int
    stride: int
    pad: int
    wrap: bool = False      # every thread of every launch runs at least two grid-stride iterations

    @property
    def ho(self) -> int:
        return out_size(self.h, self.k, self.stride, self.pad)

    @property
    def wo(self) -> int:
        return out_size(self.w, self.k, self.stride, self.pad)


# name: shape (N, C, H, W, K, stride, pad) and what it is there to reach (checked by tests/test_dwconv_dispatch_cpu.py)
CASES: Dict[str, Case] = {
    # fwd quad<1,false>, dgrad quad<1,true> (flipped filter, pad 2 - pad), wgrad quad<1>, finalize unrolled loop
    "rexnet_s1_wrap": Case(4, 96, 112, 112, 3, 1, 1, wrap=True),
    # fwd quad<2,false> with a ragged last quad (Wo = 29), the stride-2 dgrad quad at odd H / W, wgrad quad<2>
    "rexnet_s2_odd": Case(4, 144, 57, 57, 3, 2, 1),
    # dw3x3_kernel<true,2>: stride-2 data gradient with pad != 1; at pad 0 the last dx row (H = 16) is read by no output
    "s2_pad0": Case(2, 40, 16, 18, 3, 2, 0),
    "s2_pad2": Case(2, 64, 15, 15, 3, 2, 2),
    # widths below one quad: dw3x3_kernel<false,1> and <true,1>
    "narrow_s1": Case(2, 24, 9, 3, 3, 1, 1),
    # dw3x3_kernel<false,2> (Wo = 3)
    "narrow_s2": Case(2, 24, 9, 6, 3, 2, 1),
    # forward quad with pad > 1; dgrad dw3x3_kernel<true,1> (pad > 2)
    "pad3": Case(1, 32, 10, 10, 3, 1, 3),
    # runtime stride: dw3x3_kernel<false,0>, <true,0>, dw_bwd_weight_kernel<3>; the last dx column is read by no output
    "stride3": Case(2, 48, 23, 24, 3, 3, 1),
    # one channel group: cg_t = 1, rows_t = 256, one idle pixel lane in the wgrad quad kernel (256 = 3 * 85 + 1)
    "c8": Case(8, 8, 64, 64, 3, 1, 1),
    # masked channel-slab tails: 2 slabs of 21 groups (the last 20); 4 slabs of 32 groups (the last 29)
    "slab_tail_c328": Case(2, 328, 28, 28, 3, 1, 1),
    "slab_tail_c1000_s2": Case(1, 1000, 14, 14, 3, 2, 1),
    # ConvNeXt 7x7: generic forward / data gradient, dw_bwd_weight_kernel<7>, 3 slabs at C = 768
    "convnext_7x7": Case(2, 96, 56, 56, 7, 1, 3),
    "convnext_7x7_c768": Case(1, 768, 7, 7, 7, 1, 3),
    # stride 2 on the generic kernels: divisibility in the data gradient, dw_bwd_weight_kernel<5>
    "k5_s2": Case(2, 40, 17, 17, 5, 2, 2),
    "k7_s2_pad0": Case(2, 16, 20, 20, 7, 2, 0),
    # MobileOne's 1x1 branch: dw_bwd_weight_kernel<1>; generic forward / data gradient wrapping stream_grid
    "mobileone_1x1_s2": Case(4, 64, 28, 28, 1, 2, 0),
    "mobileone_1x1_wrap": Case(8, 128, 112, 112, 1, 1, 0, wrap=True),
}

# the cases the one-output 3x3 kernels and dw_bwd_weight_kernel<3> take when HB_DISABLE_DW_QUAD is set
QUAD_CASES = [name for name, cs in CASES.items() if cs.k == 3 and cs.stride in (1, 2)]


def out_size(h: int, k: int, stride: int, pad: int) -> int:
    return (h + 2 * pad - k) // stride + 1


def _cdiv(a: int, b: int) -> int:
    return -(-a // b)


def stream_grid(work: int, per_block: int, sms: int, max_waves: int = 8) -> int:
    return max(min(_cdiv(work, per_block), sms * max_waves), 1)


WGRAD_PER_SM = 2           # kWgradPerSm: row blocks per SM of the weight-gradient kernels


def scratch_doubles(c: int, k: int, sms: int) -> int:
    return S.max_blocks(c, sms, WGRAD_PER_SM) * c * (k * k + 1)


@dataclass(frozen=True)
class Launch:
    kernel: str
    total: int          # grid-stride items (pixels, quads or 8-channel vectors)
    stride: int         # items the whole grid takes per iteration (S)
    gx: int             # blocks along the item axis

    @property
    def min_iters(self) -> int:
        return self.total // self.stride

    @property
    def max_iters(self) -> int:
        return _cdiv(self.total, self.stride)


@dataclass(frozen=True)
class WgradLaunch(Launch):
    chain: int = 0      # longest per-thread fp32 accumulation chain of one dw / db element (terms)


def route_fwd(cs: Case, sms: int, quad: bool = True) -> Launch:
    n, c, ho, wo, s = cs.n, cs.c, cs.ho, cs.wo, cs.stride
    rows_t = S.geometry(c).rows_t
    if cs.k == 3 and n * ho * wo < INT_MAX:
        if quad and s in (1, 2) and wo >= 4:
            quads = n * ho * _cdiv(wo, 4)
            gx = S.grid_rows(c, quads, sms, 2, 2)
            return Launch(f"dw3x3_quad_kernel<{s},false>", quads, gx * rows_t, gx)
        gx = S.grid_rows(c, n * ho * wo, sms, 3, 4)
        return Launch(f"dw3x3_kernel<false,{s if s in (1, 2) else 0}>", n * ho * wo, gx * rows_t, gx)
    total = n * ho * wo * (c // 8)
    grid = stream_grid(total, THREADS, sms, 16)
    return Launch("dw_fwd_kernel", total, grid * THREADS, grid)


def route_dgrad(cs: Case, sms: int, quad: bool = True) -> Launch:
    n, c, h, w, s, pad = cs.n, cs.c, cs.h, cs.w, cs.stride, cs.pad
    rows_t = S.geometry(c).rows_t
    if cs.k == 3 and n * h * w < INT_MAX:
        quads = n * h * _cdiv(w, 4)
        if quad and s == 1 and w >= 4 and pad <= 2:
            gx = S.grid_rows(c, quads, sms, 2, 2)
            return Launch("dw3x3_quad_kernel<1,true>", quads, gx * rows_t, gx)
        if quad and s == 2 and pad == 1 and w >= 4:
            gx = S.grid_rows(c, quads, sms, 2, 2)
            return Launch("dw3x3_dgrad_s2_quad_kernel", quads, gx * rows_t, gx)
        gx = S.grid_rows(c, n * h * w, sms, 3, 4)
        return Launch(f"dw3x3_kernel<true,{s if s in (1, 2) else 0}>", n * h * w, gx * rows_t, gx)
    total = n * h * w * (c // 8)
    grid = stream_grid(total, THREADS, sms, 16)
    return Launch("dw_bwd_data_kernel", total, grid * THREADS, grid)


def route_wgrad(cs: Case, sms: int, quad: bool = True) -> WgradLaunch:
    """The weight-gradient kernel; ``gx`` is also the row count dw_weight_finalize_kernel folds."""
    n, c, ho, wo, s = cs.n, cs.c, cs.ho, cs.wo, cs.stride
    rows_t = S.geometry(c).rows_t
    if quad and cs.k == 3 and s in (1, 2) and rows_t >= 3:
        lanes = rows_t // 3
        quads = n * ho * _cdiv(wo, 4)
        gx = S.grid_rows(c, quads, sms, WGRAD_PER_SM, 2, lanes)
        # four outputs per quad feed each accumulator (three taps x 8 channels, and the bias column on r == 0)
        return WgradLaunch(f"dw3x3_wgrad_quad_kernel<{s}>", quads, gx * lanes, gx, 4 * _cdiv(quads, gx * lanes))
    m = n * ho * wo
    gx = S.grid_rows(c, m, sms, WGRAD_PER_SM, 8)
    return WgradLaunch(f"dw_bwd_weight_kernel<{cs.k}>", m, gx * rows_t, gx, _cdiv(m, gx * rows_t))


def finalize_unrolled(gx: int) -> bool:
    """dw_weight_finalize_kernel's four-rows-in-flight loop runs (on block lane 0 first) once gx > 96."""
    return gx > 96


def route(cs: Case, sms: int, quad: bool = True) -> Dict[str, Launch]:
    return {"fwd": route_fwd(cs, sms, quad), "dgrad": route_dgrad(cs, sms, quad), "wgrad": route_wgrad(cs, sms, quad)}


def kernels_taken(cs: Case, sms: int, quad: bool = True) -> List[str]:
    r = route(cs, sms, quad)
    out = [v.kernel for v in r.values()] + ["dw_weight_finalize_kernel"]
    if finalize_unrolled(r["wgrad"].gx):
        out.append(FINALIZE_UNROLLED)
    return out


def describe(name: str, sms: int, quad: bool = True, cs: Optional[Case] = None) -> str:
    cs = CASES[name] if cs is None else cs
    parts = [f"{d}: {v.kernel} gx={v.gx} iters {v.min_iters}..{v.max_iters}" for d, v in route(cs, sms, quad).items()]
    return f"{name} @ {sms} SMs: " + "; ".join(parts)
