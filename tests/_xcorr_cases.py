"""The NormConv2d / Add2d cases and a Python mirror of the dispatch and grid geometry of csrc/xcorr.cu, the norm path of
csrc/conv_fprop.cu and the routing of nn/_xcorr.py (no GPU).

``fwd_geo`` mirrors the grid of ``hb_xcorr2d_fwd`` (32 x 32 output tiles of (pixels L, Cout) per CTA, one grid z per
image, the K loop in 32-wide chunks); ``wgrad_geo`` the split of the atomically summed weight gradient in
``hb_xcorr2d_wgrad`` (rows m = n * L + l in 32-row chunks, ``cps`` chunks per split, one split per grid z);
``dgrad_uncovered`` the input pixels ``hb_add2d_dgrad`` finds no output window for; ``route`` the choice of
``_XcorrFn.forward``; ``tc_launch`` the Cout tile rule of ``fprop_launch`` with the patch-normalisation epilogue (no
statistics, no dual output, so the wide tiles are open to it). The SM count sizes the weight-gradient split and the
wide-tile condition, so both take it as an argument (H100 SXM: 132, H100 PCIe: 114)."""
from dataclasses import dataclass
from typing import Dict, List, Set, Tuple

TL = TC = TK = 32           # xcorr.cu tile sizes: pixels, output channels, reduction chunk
BM = 128                    # conv_fprop.cu pixel tile
MAX_GRID_YZ = 65535


def _cdiv(a: int, b: int) -> int:
    return -(-a // b)


def round_up(v: int, m: int) -> int:
    return _cdiv(v, m) * m


@dataclass(frozen=True)
class Case:
    n: int
    cin: int
    h: int
    w: int
    cout: int
    kh: int
    kw: int
    stride: int = 1
    pad: int = 0
    dil: int = 1

    @property
    def ho(self) -> int:
        return (self.h + 2 * self.pad - self.dil * (self.kh - 1) - 1) // self.stride + 1

    @property
    def wo(self) -> int:
        return (self.w + 2 * self.pad - self.dil * (self.kw - 1) - 1) // self.stride + 1

    @property
    def k(self) -> int:
        return self.cin * self.kh * self.kw

    @property
    def l(self) -> int:  # noqa: E743
        return self.ho * self.wo

    @property
    def m(self) -> int:
        return self.n * self.l


# fp32 CUDA-core kernels: every case runs the forward in both modes (norm_conv, adder) with and without normalisation,
# the weight gradient in the same four configurations, and the adder data gradient.
# name: shape and what it is there to reach (checked by tests/test_xcorr_dispatch_cpu.py)
CASES: Dict[str, Case] = {
    # RGB stem: K = 27 < 32 (one partial K chunk); Cout = 40: two Cout tiles, the second 8 wide; L = 143: a ragged L
    # tile; wgrad: 9 single-chunk splits, the last one 30 rows, chunk 4 straddles images 0 and 1
    "rgb_k27": Case(2, 3, 13, 11, 40, 3, 3, 1, 1),
    # K = 72 (3 chunks, the last 8 wide); M = 1860: 59 chunks in 30 splits of 2 (cps = 2 at 132 and 114 SMs), the last
    # split one partial chunk; chunk 29 straddles images 0 and 1
    "k72_cps2": Case(2, 8, 31, 30, 40, 3, 3, 1, 1),
    # K = 64 and Cout = 64: no ragged K or Cout tile (only L = 81 is ragged)
    "k64_1x1": Case(2, 64, 9, 9, 64, 1, 1),
    # stride 2, pad 0: the last input row (15) is read by no window; K = 36, Cout = 24
    "s2_pad0": Case(2, 4, 16, 15, 24, 3, 3, 2, 0),
    # stride 3, pad 0: rows 15, 16 and columns 18, 19 are read by no window
    "s3_pad0": Case(2, 5, 17, 20, 16, 3, 3, 3, 0),
    # stride 2, dilation 2, pad 2: every tap lands on an even row / column, the odd ones are read by no window
    "s2_dil2": Case(2, 6, 15, 14, 36, 3, 3, 2, 2, 2),
    # dilation 2 at stride 1: every pixel is read, through windows two pixels apart
    "dil2": Case(1, 8, 12, 12, 32, 3, 3, 1, 2, 2),
    # a 3 x 1 filter with the symmetric padding 1: the padded columns make all-zero windows; _XcorrFn routes NormConv2d
    # with it to the fp32 kernel
    "rect_3x1": Case(2, 16, 10, 9, 48, 3, 1, 1, 1),
}

# tensor-core NormConv2d: hb_patch_stats_bf16, then hb_conv2d_fused_bf16 with the norm_* epilogue
TC_CASES: Dict[str, Case] = {
    # Cin = 3 (channels padded to 8, k_logical = 27), Cout = 24 (padded to 32, then sliced): one narrow 32-column tile
    "tc_rgb_stem": Case(2, 3, 20, 18, 24, 3, 3, 1, 1),
    # narrow whole 64-column tile, stride 2 on odd sizes
    "tc_narrow64_s2": Case(2, 16, 33, 29, 64, 3, 3, 2, 1),
    # dilation 2: border rows and columns of windows are two pixels into the padding
    "tc_dil2": Case(2, 8, 19, 17, 48, 3, 3, 1, 2, 2),
    # Cout = 144 at small M (4 pixel tiles): 128-column tiles, the second one masked to 16 columns
    "tc_masked144": Case(1, 16, 20, 20, 144, 3, 3, 1, 1),
    # large M (>= 132 pixel tiles per Cout tile): 192-column tiles (384 = 2 x 192, 256 does not divide it)
    "tc_wide192": Case(1, 8, 92, 92, 384, 3, 3, 1, 1),
    # large M, Cout = 256: one 256-column tile
    "tc_wide256": Case(2, 8, 96, 96, 256, 3, 3, 1, 1),
    # a 1 x 1 filter is never given a wide tile: Cout = 192 at large M takes two 96-column tiles
    "tc_1x1_cout192": Case(2, 16, 96, 96, 192, 1, 1),
}


# ---------------------------------------------------------------------------------------------------------------------
# hb_xcorr2d_fwd
# ---------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class FwdGeo:
    grid: Tuple[int, int, int]      # (L tiles, Cout tiles, N)
    k_chunks: int                   # trips of the 32-wide K loop
    ragged: Tuple[str, ...]         # dimensions whose last tile / chunk is partial: "L", "Cout", "K"


def fwd_geo(cs: Case) -> FwdGeo:
    ragged = tuple(d for d, v, t in (("L", cs.l, TL), ("Cout", cs.cout, TC), ("K", cs.k, TK)) if v % t)
    return FwdGeo((_cdiv(cs.l, TL), _cdiv(cs.cout, TC), cs.n), _cdiv(cs.k, TK), ragged)


def fwd_kernels(cs: Case) -> List[str]:
    """The instantiations one case runs: both modes, each with and without the fp32 patch statistics."""
    return [f"xcorr_fwd_kernel<{adder}>" + ("+patch_stats_kernel" if norm else "")
            for adder in ("false", "true") for norm in (False, True)]


# ---------------------------------------------------------------------------------------------------------------------
# hb_xcorr2d_wgrad
# ---------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class WgradGeo:
    tiles: int                      # (K tiles) x (Cout tiles): CTAs per split
    splits: int                     # grid z
    cps: int                        # 32-row chunks per split
    chunks: int
    last_rows: int                  # rows m of the last split
    straddling: Tuple[int, ...]     # chunks whose rows belong to two images (m crosses a multiple of L)

    @property
    def last_partial(self) -> bool:
        return self.last_rows < self.cps * TL

    @property
    def chain(self) -> int:
        """Longest fp32 accumulation chain of one dw element: one thread's rows, then one atomicAdd per split."""
        return self.cps * TL + self.splits


def wgrad_geo(cs: Case, sms: int) -> WgradGeo:
    m = cs.m
    chunks = _cdiv(m, TL)
    tiles = _cdiv(cs.k, TK) * _cdiv(cs.cout, TC)
    splits = max(min(_cdiv(sms * 2, tiles), chunks), 1)
    splits = min(splits, MAX_GRID_YZ)
    cps = _cdiv(chunks, splits)
    gz = _cdiv(chunks, cps)
    straddle = tuple(j for j in range(chunks) if (j * TL) // cs.l != (min(j * TL + TL, m) - 1) // cs.l)
    return WgradGeo(tiles, gz, cps, chunks, m - (gz - 1) * cps * TL, straddle)


def wgrad_paths(cs: Case, sms: int) -> Set[str]:
    g = wgrad_geo(cs, sms)
    out = {"wgrad_cps>1" if g.cps > 1 else "wgrad_cps=1"}
    if g.splits > 1:
        out.add("wgrad_several_splits")
    if g.last_partial:
        out.add("wgrad_partial_last_split")
    if g.straddling:
        out.add("wgrad_straddling_chunk")
    return out


# ---------------------------------------------------------------------------------------------------------------------
# hb_add2d_dgrad
# ---------------------------------------------------------------------------------------------------------------------
def _uncovered(size: int, out: int, k: int, stride: int, pad: int, dil: int) -> List[int]:
    read = {o * stride - pad + r * dil for o in range(out) for r in range(k)}
    return [i for i in range(size) if i not in read]


def dgrad_uncovered(cs: Case) -> Tuple[List[int], List[int]]:
    """(input rows, input columns) no output window reads: their data gradient is exactly 0."""
    return (_uncovered(cs.h, cs.ho, cs.kh, cs.stride, cs.pad, cs.dil),
            _uncovered(cs.w, cs.wo, cs.kw, cs.stride, cs.pad, cs.dil))


def dgrad_paths(cs: Case) -> Set[str]:
    rows, cols = dgrad_uncovered(cs)
    out = {f"dgrad_stride{cs.stride}"}
    if rows or cols:
        out.add(f"dgrad_stride{cs.stride}_uncovered")
    if cs.dil > 1:
        out.add("dgrad_dilated")
    return out


# ---------------------------------------------------------------------------------------------------------------------
# _XcorrFn routing and the tensor-core Cout tile rule
# ---------------------------------------------------------------------------------------------------------------------
def route(cs: Case, mode: int, normalize: bool) -> str:
    """The forward kernel _XcorrFn.forward takes (HB_NORMCONV_FP32 unset)."""
    if mode == 0 and normalize and cs.kh == cs.kw:
        return "tensor_cores"
    return f"xcorr_fwd_kernel<{'true' if mode == 1 else 'false'}>"


@dataclass(frozen=True)
class TcLaunch:
    cin_p: int                      # channels of the packed bf16 input (a multiple of 8)
    cout_p: int                     # rows of the packed filter (a multiple of 16)
    bn: int                         # Cout tile
    m_tiles: int
    kind: str


def cout_tile(cout: int, taps: int, m_tiles: int, grid: int) -> int:
    """BN of fprop_launch for a single-output launch without statistics."""
    if cout <= 128:
        return cout
    bn = next((c for c in range(128, 63, -16) if cout % c == 0), 128)
    wide = 0 if taps == 1 else cout if cout <= 256 else 256 if cout % 256 == 0 else 192 if cout % 192 == 0 else 0
    if wide and m_tiles * (cout // wide) >= grid:
        bn = wide
    return bn


def tc_launch(cs: Case, sms: int, num_ctas: int = 0) -> TcLaunch:
    cin_p, cout_p = round_up(cs.cin, 8), round_up(cs.cout, 16)
    m_tiles = _cdiv(cs.m, BM)
    grid = min(num_ctas if num_ctas > 0 else sms, 4 * sms)
    bn = cout_tile(cout_p, cs.kh * cs.kw, m_tiles, grid)
    if bn > 128:
        kind = f"wide{bn}"
    elif cout_p <= 128:
        kind = "narrow_whole"
    elif cout_p % bn:
        kind = "narrow_masked"
    elif cs.kh * cs.kw == 1 and cout_tile(cout_p, 9, m_tiles, grid) > 128:
        kind = "narrow_1x1_at_wide_size"
    else:
        kind = "narrow_split"
    return TcLaunch(cin_p, cout_p, bn, m_tiles, kind)


def tc_paths(cs: Case, sms: int) -> Set[str]:
    t = tc_launch(cs, sms)
    out = {t.kind}
    if t.cin_p != cs.cin:
        out.add("cin_padded")
    if t.cout_p != cs.cout:
        out.add("cout_padded_sliced")
    return out


def describe(name: str, sms: int) -> str:
    if name in TC_CASES:
        t = tc_launch(TC_CASES[name], sms)
        return f"{name} @ {sms} SMs: BN={t.bn} ({t.kind}), {t.m_tiles} pixel tiles, Cin {t.cin_p}, Cout {t.cout_p}"
    cs = CASES[name]
    f, g = fwd_geo(cs), wgrad_geo(cs, sms)
    return (f"{name} @ {sms} SMs: fwd grid {f.grid}, {f.k_chunks} K chunks, ragged {f.ragged}; wgrad {g.tiles} tiles x "
            f"{g.splits} splits of {g.cps} chunks (last {g.last_rows} rows), straddling {g.straddling}")
