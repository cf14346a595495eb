"""The convolution kernels per element (tests/_bounds.py), at forced grid sizes and at the tile edges real layers reach.

Forced grids. Every convolution kernel is persistent: a CTA walks its tiles (pixel tiles of one Cout tile, row-window
tiles, weight-gradient units) carrying its ring stage / phase, its staging tile and its statistics registers from tile to
tile. With one CTA per SM the small test shapes give each CTA one tile, so each case here also runs at num_ctas = 1, 2, 3
and 7, where every CTA walks many tiles and the ring phase wraps in the middle of a tile. Each element is computed by one
CTA in the same K order whatever the grid, so every output must be bit-identical to the default grid's (the wide Cout
tiles, taken on small shapes only when the grid is small, included). Statistics launches must report 2 slots per CTA of
one Cout tile, their slots must add up to the sums of the stored output, and a repeat must give the same bits.

Edges. Output widths with a masked Cout tail (176, 304, 368, 848: ReXNet's padded widths), weight gradients with a
partial last Cin tile (176, 368, 840), the row-window kernel at its width limits (W = 8 and 126), at H = 1 and 2 and with
a partial channel block, generic filters (5x5, 7x7, dilation 2 and 3, pad 0), stride 2 on odd sizes, and M around one
128-pixel tile. Everything goes through the C ABI."""
import ctypes

import pytest
import torch

from holocron_b200._lib import ConvArgs, lib, ptr, stream_ptr

from _bounds import FP32_BITS, assert_within, check_stats, conv_ref, dgrad_ref, epilogue_ref, ulp, wgrad_ref

pytestmark = pytest.mark.gpu
GRIDS = [0, 1, 2, 3, 7]          # 0 = one CTA per SM, run first: the other grids must reproduce its bits


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def bf16(*shape, scale=1.0):
    return (torch.randn(*shape) * scale).bfloat16()


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous().cuda()


def nchw(t):
    return t.permute(0, 3, 1, 2).cpu()


def krsc(w):
    return w.permute(0, 2, 3, 1).contiguous().cuda()


def _out_size(h, k, stride, pad, dil):
    return (h + 2 * pad - dil * (k - 1) - 1) // stride + 1


def fused(x, w, cout, k, stride=1, pad=0, dil=1, *, bias=None, residual=None, act=0, num_ctas=0, xe=None, we=None, w2=None,
          stats=False):
    """One hb_conv2d_fused_bf16 launch. x: NHWC bf16 (cuda), w: KRSC bf16; returns (y, y2, parts, parts2, slots), NHWC."""
    n, h, wd, cin = x.shape
    ho, wo = _out_size(h, k, stride, pad, dil), _out_size(wd, k, stride, pad, dil)
    nan = float("nan")
    y = torch.full((n, ho, wo, cout), nan, device="cuda", dtype=torch.bfloat16)
    y2 = torch.full_like(y, nan) if w2 is not None else None
    cap = lib().hb_conv_stat_slots_max()
    parts = torch.full((cap, cout, 2), nan, device="cuda") if stats else None
    parts2 = torch.full((cap, cout, 2), nan, device="cuda") if stats and w2 is not None else None
    a = ConvArgs()
    a.x, a.w, a.y = x.data_ptr(), w.data_ptr(), y.data_ptr()
    a.bias = 0 if bias is None else bias.data_ptr()
    a.residual = 0 if residual is None else residual.data_ptr()
    a.N, a.H, a.W, a.Cin, a.Cout, a.R, a.S = n, h, wd, cin, cout, k, k
    a.stride, a.pad, a.dil, a.act, a.num_ctas = stride, pad, dil, act, num_ctas
    if xe is not None:
        a.xe, a.we, a.Ce = xe.data_ptr(), we.data_ptr(), xe.shape[-1]
    if w2 is not None:
        a.w2, a.y2 = w2.data_ptr(), y2.data_ptr()
    if stats:
        a.stats = parts.data_ptr()
        if parts2 is not None:
            a.stats2 = parts2.data_ptr()
    slots = ctypes.c_int(-1)
    rc = lib().hb_conv2d_fused_bf16(ctypes.byref(a), ctypes.byref(slots), stream_ptr())
    assert rc == 0, rc
    torch.cuda.synchronize()
    return y, y2, parts, parts2, slots.value


def narrow_n_tiles(cout, dual=False):
    """Cout tiles of a statistics launch (narrow rule of conv_fprop.cu: whole Cout up to the limit, else the largest
    multiple of 16 in [64, limit] dividing it, else the limit with a masked tail)."""
    lim = 64 if dual else 128
    bn = cout
    if cout > lim:
        bn = next((c for c in range(lim, 63, -16) if cout % c == 0), lim)
    return (cout + bn - 1) // bn


def fprop_slots(num_ctas, n_tiles, m_tiles):
    grid = min(num_ctas if num_ctas > 0 else _sms(), 4 * _sms())
    return 2 * min(max(grid // n_tiles, 1), m_tiles)


# ---------------------------------------------------------------------------------------------------------------------
# forced grids: hb_conv2d_fused_bf16 on the generic implicit-GEMM kernel
# ---------------------------------------------------------------------------------------------------------------------
FPROP_GRID_CASES = {
    # name: (N, H, Cin, Cout, k, stride, options)
    "narrow_3x3_cin144": (2, 20, 144, 96, 3, 1, {}),                    # 7 pixel tiles, 27 K blocks per tile
    "wide_3x3_cout192": (2, 24, 64, 192, 3, 1, {}),                     # small grids take the 192-column tile
    "wide_3x3_s2_cout256_odd": (2, 47, 64, 256, 3, 2, {}),              # 256-column tile, stride 2, odd H/W
    "dual_output_stats": (2, 18, 48, 64, 3, 1, {"dual": True, "stats": True}),
    "kext_ce40_residual": (2, 20, 48, 80, 3, 1, {"ce": 40, "residual": True}),
    "bias_relu_1x1_cout176": (2, 19, 72, 176, 1, 1, {"bias": True, "relu": True}),
    "bias_relu_residual_3x3": (2, 17, 136, 48, 3, 1, {"bias": True, "relu": True, "residual": True}),
    "stats_bias_3x3_cin144": (2, 20, 144, 112, 3, 1, {"bias": True, "stats": True}),
    "stats_1x1_cout304": (1, 30, 64, 304, 1, 1, {"stats": True}),
}


@pytest.mark.parametrize("name", list(FPROP_GRID_CASES))
def test_fprop_forced_grids(name):
    n, h, cin, cout, k, stride, o = FPROP_GRID_CASES[name]
    torch.manual_seed(len(name))
    pad = k // 2
    x = bf16(n, cin, h, h)
    w = bf16(cout, cin, k, k, scale=(cin * k * k) ** -0.5)
    bias = torch.randn(cout) if o.get("bias") else None
    acc, abs_sum = conv_ref(x, w, bias, stride, pad)
    ho = acc.shape[2]
    xe = we = w2 = res = None
    if o.get("ce"):
        xe = bf16(n, o["ce"], ho, ho)
        we = bf16(cout, o["ce"], 1, 1, scale=o["ce"] ** -0.5)
        a2, s2 = conv_ref(xe, we)
        acc, abs_sum = acc + a2, abs_sum + s2
    if o.get("residual"):
        res = bf16(n, cout, ho, ho)
    ref, abs_sum, slack = epilogue_ref(acc, abs_sum, res, o.get("relu", False))
    if o.get("dual"):
        w2 = bf16(cout, cin, 1, 1, scale=cin ** -0.5)
        ref2, abs2 = conv_ref(x, w2, None, stride, 0)
    stats = o.get("stats", False)
    m_tiles = (n * ho * ho + 127) // 128
    n_tiles = narrow_n_tiles(cout, w2 is not None)
    args = dict(bias=None if bias is None else bias.cuda(), residual=None if res is None else nhwc(res),
                act=1 if o.get("relu") else 0, xe=None if xe is None else nhwc(xe), we=None if we is None else krsc(we),
                w2=None if w2 is None else krsc(w2), stats=stats)
    xg, wg = nhwc(x), krsc(w)
    base = None
    for g in GRIDS:
        what = f"{name} num_ctas={g}"
        y, y2, parts, parts2, slots = fused(xg, wg, cout, k, stride, pad, num_ctas=g, **args)
        assert_within(nchw(y), ref, abs_sum, what, slack=slack)
        if y2 is not None:
            assert_within(nchw(y2), ref2, abs2, what + " y2")
        if stats:
            assert slots == fprop_slots(g, n_tiles, m_tiles), what
            check_stats(y, parts, slots, what)
            if parts2 is not None:
                check_stats(y2, parts2, slots, what + " y2")
            again = fused(xg, wg, cout, k, stride, pad, num_ctas=g, **args)
            assert again[4] == slots and torch.equal(again[2][:slots], parts[:slots]), what + ": statistics not repeatable"
            if parts2 is not None:
                assert torch.equal(again[3][:slots], parts2[:slots]), what + ": statistics y2 not repeatable"
        if base is None:
            base = (y, y2)
        else:
            assert torch.equal(y, base[0]), what + ": output differs from the default grid's"
            assert y2 is None or torch.equal(y2, base[1]), what + ": y2 differs from the default grid's"


# ---------------------------------------------------------------------------------------------------------------------
# forced grids: row-window kernel (conv_rows.cu), plain, with statistics, and hb_conv3x3_accum_bf16
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stats", [False, True])
def test_rows_forced_grids(stats):
    # W = 30: 4 output rows per 128-pixel sub-tile; H = 62 is not a multiple of the tile rows (12 or 16 here)
    n, h, w, cin, cout = 2, 62, 30, 48, 64 if not stats else 32
    torch.manual_seed(11 + stats)
    x = bf16(n, cin, h, w)
    wt = bf16(cout, cin, 3, 3, scale=(9 * cin) ** -0.5)
    ref, abs_sum = conv_ref(x, wt, None, 1, 1)
    xg, wg = nhwc(x), krsc(wt)
    base = None
    for g in GRIDS:
        what = f"rows stats={stats} num_ctas={g}"
        y, _, parts, _, slots = fused(xg, wg, cout, 3, 1, 1, num_ctas=g, stats=stats)
        assert_within(nchw(y), ref, abs_sum, what)
        if stats:
            if g:
                assert slots == 2 * g, what          # the shape has more row-window tiles than 7
            else:
                assert slots % 2 == 0 and 2 <= slots <= 2 * _sms(), what
            check_stats(y, parts, slots, what)
            again = fused(xg, wg, cout, 3, 1, 1, num_ctas=g, stats=True)
            assert again[4] == slots and torch.equal(again[2][:slots], parts[:slots]), what + ": statistics not repeatable"
        if base is None:
            base = y
        else:
            assert torch.equal(y, base), what + ": output differs from the default grid's"


@pytest.mark.parametrize("nextra", [0, 1, 2])
def test_accum_forced_grids(nextra):
    n, h, w, cin, cout = 2, 41, 22, 32, 48
    torch.manual_seed(20 + nextra)
    x = bf16(n, cin, h, w)
    wt = bf16(cout, cin, 3, 3, scale=(9 * cin) ** -0.5)
    ref, abs_sum = conv_ref(x, wt, None, 1, 1)
    xes = [bf16(n, cin, h, w) for _ in range(nextra)]
    wes = [bf16(cout, cin, 1, 1, scale=cin ** -0.5) for _ in range(nextra)]
    for xe, we in zip(xes, wes):
        r2, s2 = conv_ref(xe, we)
        ref, abs_sum = ref + r2, abs_sum + s2
    xg, wg = nhwc(x), krsc(wt)
    eg = [nhwc(t) for t in xes] + [None] * (2 - nextra)
    weg = [krsc(t) for t in wes] + [None] * (2 - nextra)
    base = None
    for g in GRIDS:
        what = f"accum nextra={nextra} num_ctas={g}"
        y = torch.full((n, h, w, cout), float("nan"), device="cuda", dtype=torch.bfloat16)
        rc = lib().hb_conv3x3_accum_bf16(ptr(xg), ptr(wg), ptr(eg[0]), ptr(weg[0]), ptr(eg[1]), ptr(weg[1]), nextra, ptr(y),
                                         n, h, w, cin, cout, g, stream_ptr())
        assert rc == 0, (what, rc)
        torch.cuda.synchronize()
        assert_within(nchw(y), ref, abs_sum, what)
        if base is None:
            base = y
        else:
            assert torch.equal(y, base), what + ": output differs from the default grid's"


# ---------------------------------------------------------------------------------------------------------------------
# forced grids: parity-class stride-2 data gradient (hb_conv2d_dgrad_s2_bf16)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with1x1", [False, True])
def test_dgrad_s2_forced_grids(with1x1):
    n, h, c, cd = 2, 45, 48, 64          # dy [2, 23, 23, 48] -> dx [2, 45, 45, 64]; class (0, 0) has 9 pixel tiles
    torch.manual_seed(30 + with1x1)
    ho = (h - 1) // 2 + 1
    w3 = bf16(c, cd, 3, 3, scale=(9 * cd) ** -0.5)
    w1 = bf16(c, cd, 1, 1, scale=cd ** -0.5)
    dy3, dy1 = bf16(n, c, ho, ho), bf16(n, c, ho, ho)
    ref3, abs_sum = dgrad_ref((n, cd, h, h), w3, dy3, 2, 1)
    ref, slack = ref3, None
    if with1x1:
        # the 1x1 branch is stored first (bf16) and class (0, 0) of the 3x3 part, rounded to bf16, is added onto it
        ref1, abs1 = dgrad_ref((n, cd, h, h), w1, dy1, 2, 0)
        ref, abs_sum = ref3 + ref1, abs_sum + abs1
        cls00 = torch.zeros_like(ref, dtype=torch.bool)
        cls00[:, :, ::2, ::2] = True
        slack = torch.where(cls00, 0.5 * (ulp(ref1) + ulp(ref3)), torch.zeros_like(ref))
    wcls = torch.empty(9 * cd * c, device="cuda", dtype=torch.bfloat16)
    assert lib().hb_pack_dgrad_s2_weights(ptr(w3.float().permute(0, 2, 3, 1).contiguous().cuda()), ptr(wcls), c, cd, cd, c,
                                          stream_ptr()) == 0
    wd1 = w1[:, :, 0, 0].t().contiguous().reshape(cd, 1, 1, c).cuda()
    d3, d1 = nhwc(dy3), nhwc(dy1)
    base = None
    for g in GRIDS:
        what = f"dgrad_s2 with1x1={with1x1} num_ctas={g}"
        dx = torch.full((n, h, h, cd), float("nan"), device="cuda", dtype=torch.bfloat16)
        rc = lib().hb_conv2d_dgrad_s2_bf16(ptr(d3), ptr(wcls), ptr(d1 if with1x1 else None), ptr(wd1 if with1x1 else None),
                                           ptr(dx), n, h, h, ho, ho, c, cd, g, stream_ptr())
        assert rc == 0, (what, rc)
        torch.cuda.synchronize()
        assert_within(nchw(dx), ref, abs_sum, what, slack=slack)
        if base is None:
            base = dx
        else:
            assert torch.equal(dx, base), what + ": output differs from the default grid's"


# ---------------------------------------------------------------------------------------------------------------------
# forced grids: weight gradients (generic split-K kernel, row-window kernel, one-pass RepVGG kernel)
# ---------------------------------------------------------------------------------------------------------------------
WGRAD_GRIDS = [1, 2, 7, 0]
WGRAD_CASES = {
    # name: (N, H, W, Cin, Cout, k, stride, pad)
    "generic_1x1": (2, 32, 32, 64, 96, 1, 1, 0),       # one unit: grid 1 stores, grids 2 / 7 / 0 split the pixels
    "generic_3x3_s2": (2, 33, 33, 48, 32, 3, 2, 1),
    "rows_3x3": (2, 40, 22, 48, 16, 3, 1, 1),          # row-window kernel (one CTA group)
    "rows_3x3_cin72": (2, 24, 30, 72, 32, 3, 1, 1),    # 4 CTA groups: grids 1 and 2 run the generic kernel
}


def _wgrad(x, dy, dw, ws, wsb, n, h, w, cin, cout, k, stride, pad, g):
    rc = lib().hb_conv2d_wgrad_bf16(ptr(x), ptr(dy), ptr(dw), ptr(ws), wsb, n, h, w, cin, cout, k, k, stride, pad, 1, g,
                                    stream_ptr())
    assert rc == 0, rc
    torch.cuda.synchronize()


@pytest.mark.parametrize("name", list(WGRAD_CASES))
def test_wgrad_forced_grids(name):
    n, h, w, cin, cout, k, stride, pad = WGRAD_CASES[name]
    torch.manual_seed(40 + len(name))
    x = bf16(n, cin, h, w)
    ho, wo = _out_size(h, k, stride, pad, 1), _out_size(w, k, stride, pad, 1)
    dy = bf16(n, cout, ho, wo)
    ref, abs_sum = wgrad_ref(x, dy, k, stride, pad)
    ref, abs_sum = ref.permute(0, 2, 3, 1), abs_sum.permute(0, 2, 3, 1)
    xg, dg = nhwc(x), nhwc(dy)
    for g in WGRAD_GRIDS:
        what = f"{name} num_ctas={g}"
        wsb = lib().hb_conv2d_wgrad_workspace_bytes(n, h, w, cin, cout, k, k, stride, pad, 1, g)
        outs = []
        for _ in range(2):
            ws = torch.empty(max(wsb // 4, 1), device="cuda") if wsb else None
            dw = torch.full((cout, k, k, cin), float("nan"), device="cuda")
            _wgrad(xg, dg, dw, ws, wsb, n, h, w, cin, cout, k, stride, pad, g)
            outs.append(dw)
        assert_within(outs[0].cpu(), ref, abs_sum, what, bits=FP32_BITS)
        assert torch.equal(outs[0], outs[1]), what + ": not bit-reproducible"
    # no workspace: more than one pixel range is accumulated with fp32 atomics
    dw = torch.full((cout, k, k, cin), float("nan"), device="cuda")
    _wgrad(xg, dg, dw, None, 0, n, h, w, cin, cout, k, stride, pad, 0)
    assert_within(dw.cpu(), ref, abs_sum, name + " atomics", bits=FP32_BITS)


def test_repvgg_wgrad_forced_grids():
    n, h, w, cin, cout = 2, 40, 22, 48, 16
    torch.manual_seed(50)
    x, dy3, dy1 = bf16(n, cin, h, w), bf16(n, cout, h, w), bf16(n, cout, h, w)
    r3, a3 = wgrad_ref(x, dy3, 3, 1, 1)
    r1, a1 = wgrad_ref(x, dy1, 1)
    xg, d3, d1 = nhwc(x), nhwc(dy3), nhwc(dy1)
    for g in WGRAD_GRIDS:
        what = f"repvgg wgrad num_ctas={g}"
        wsb = lib().hb_repvgg_wgrad_workspace_bytes(n, h, w, cin, cout, g)
        assert wsb > 0, what
        outs = []
        for _ in range(2):
            ws = torch.empty(wsb // 4, device="cuda")
            dw = torch.full((cout * 10 * cin,), float("nan"), device="cuda")
            rc = lib().hb_repvgg_wgrad_bf16(ptr(xg), ptr(d3), ptr(d1), ptr(dw), ptr(ws), wsb, n, h, w, cin, cout, g, stream_ptr())
            assert rc == 0, (what, rc)
            torch.cuda.synchronize()
            outs.append(dw)
        dw = outs[0].cpu()
        assert_within(dw[:cout * 9 * cin].view(cout, 3, 3, cin), r3.permute(0, 2, 3, 1), a3.permute(0, 2, 3, 1), what + " dW3",
                      bits=FP32_BITS)
        assert_within(dw[cout * 9 * cin:].view(cout, 1, 1, cin), r1.permute(0, 2, 3, 1), a1.permute(0, 2, 3, 1), what + " dW1",
                      bits=FP32_BITS)
        assert torch.equal(outs[0], outs[1]), what + ": not bit-reproducible"


# ---------------------------------------------------------------------------------------------------------------------
# edges
# ---------------------------------------------------------------------------------------------------------------------
def _check_forward(n, h, w, cin, cout, k, stride, pad, dil=1, bias=True, stats=False, seed=0, what=""):
    torch.manual_seed(seed)
    x = bf16(n, cin, h, w)
    wt = bf16(cout, cin, k, k, scale=(cin * k * k) ** -0.5)
    b = torch.randn(cout) if bias else None
    ref, abs_sum = conv_ref(x, wt, b, stride, pad, dil)
    xg = x.permute(0, 2, 3, 1).contiguous().cuda()
    y, _, parts, _, slots = fused(xg, krsc(wt), cout, k, stride, pad, dil, bias=None if b is None else b.cuda(), stats=stats)
    assert_within(nchw(y), ref, abs_sum, what)
    if stats:
        check_stats(y, parts, slots, what)


@pytest.mark.parametrize("stats", [False, True])
@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("cout", [176, 304, 368, 848])
def test_masked_cout_tail(cout, k, stats):
    # no multiple of 16 in 64..128 divides these widths: 128-column tiles with a partly masked last one
    _check_forward(1, 12, 12, 64, cout, k, 1, k // 2, stats=stats, seed=cout + k, what=f"Cout {cout} {k}x{k} stats={stats}")


@pytest.mark.parametrize("k,stride", [(1, 1), (3, 2)])
@pytest.mark.parametrize("cin", [176, 368, 840])
def test_wgrad_partial_cin_tile(cin, k, stride):
    # Cin tiles of 128 channels plus a partial last one (48, 112 and 72 channels)
    n, h, cout = 2, 15, 32
    pad = k // 2
    torch.manual_seed(cin + k)
    x = bf16(n, cin, h, h)
    ho = _out_size(h, k, stride, pad, 1)
    dy = bf16(n, cout, ho, ho)
    ref, abs_sum = wgrad_ref(x, dy, k, stride, pad)
    wsb = lib().hb_conv2d_wgrad_workspace_bytes(n, h, h, cin, cout, k, k, stride, pad, 1, 0)
    ws = torch.empty(max(wsb // 4, 1), device="cuda") if wsb else None
    dw = torch.full((cout, k, k, cin), float("nan"), device="cuda")
    _wgrad(nhwc(x), nhwc(dy), dw, ws, wsb, n, h, h, cin, cout, k, stride, pad, 0)
    assert_within(dw.cpu(), ref.permute(0, 2, 3, 1), abs_sum.permute(0, 2, 3, 1), f"wgrad Cin {cin}", bits=FP32_BITS)


ROWS_EDGES = [(w, h, 72) for w in (8, 62, 126) for h in (1, 2, 37)] + [(w, 37, 120) for w in (8, 62, 126)]


@pytest.mark.parametrize("w,h,cin", ROWS_EDGES)
def test_rows_kernel_limits(w, h, cin):
    # 8 <= W <= 126: W = 126 fills a 128-pixel sub-tile with one output row, W = 8 packs 12; H = 37 is not a multiple
    # of the tile rows; Cin 72 / 120: a partial second channel block
    _check_forward(2, h, w, cin, 32, 3, 1, 1, seed=w + h + cin, what=f"rows W={w} H={h} Cin={cin}")


@pytest.mark.parametrize("k,dil,pad", [(5, 1, 2), (7, 1, 3), (3, 2, 2), (3, 3, 3), (3, 1, 0)])
def test_generic_filters(k, dil, pad):
    _check_forward(2, 19, 19, 40, 48, k, 1, pad, dil, seed=k * 10 + dil, what=f"{k}x{k} dil {dil} pad {pad}")


@pytest.mark.parametrize("k,h,w", [(3, 21, 21), (1, 21, 21), (3, 21, 15), (1, 15, 21)])
def test_stride2_odd_sizes(k, h, w):
    _check_forward(2, h, w, 48, 64, k, 2, k // 2, seed=h + w + k, what=f"{k}x{k} stride 2 on {h}x{w}")


@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("m", [1, 127, 128, 129])
def test_pixels_around_one_tile(m, k):
    _check_forward(1, 1, m, 64, 80, k, 1, k // 2, seed=m + k, what=f"M={m} {k}x{k}")
