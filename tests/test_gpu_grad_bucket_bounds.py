"""The gradient-bucket plumbing of the training step, per element and bit for bit.

a. ``hb_conv2d_wgrad_acc_bf16`` / ``hb_repvgg_wgrad_acc_bf16`` on every path of tests/_grad_bucket_oracle.py's case tables:
   the accumulating form equals torch's fp32 ``prior + overwriting form`` bit for bit (the reduction adds the prior last),
   the overwriting form is within the fp32 bound of an fp64 weight gradient, and a refused shape (801) touches nothing.
b. The filter packing kernels, single and multi-tensor, bit for bit against the restatement, and the ``_PackTable`` path
   after an in-place parameter update.
c. ``hb_grad_clip_norm`` per element against ``clip_grad_norm_``'s arithmetic, NaN and inf norms included.
d. A ``GradBucket(direct=True)`` model and a ``direct=False`` one give bit-identical gradients over two accumulated
   micro-batches, on each of the six routes a parameter gradient can take into the bucket.
e. A graphed training step (``GraphedTrainStep``) and the same step launched eagerly keep bit-identical losses,
   parameters, optimizer states and BatchNorm buffers, and the graph re-packs the filters from the current masters.

Outputs are NaN-filled and guarded by NaN-payload words that must come back with the same bits."""
import ctypes
import gc

import numpy as np
import pytest
import torch
import torch.nn.functional as TF

import _grad_bucket_oracle as O
import holocron_b200 as hb
from _bounds import FP32_BITS, assert_within, wgrad_ref
from holocron_b200._lib import lib, ptr, stream_ptr
from holocron_b200.distributed import GradBucket
from holocron_b200.graphs import GraphedTrainStep
from holocron_b200.models.classification.repvgg import RepBlock
from holocron_b200.nn import _fused

pytestmark = pytest.mark.gpu
DEV = "cuda"
GUARD = 16                              # guard elements at least, before, between and after the views
GUARD_BITS = 0x7FC0DEAD                 # an fp32 NaN payload no kernel writes
GUARD_BITS16 = 0x7FAD                   # a bf16 NaN payload no kernel writes
MISALIGNED, INVALID = 716, 1


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _nhwc_bf16(n, c, h, w, gen):
    return torch.randn(n, c, h, w, device=DEV, generator=gen).bfloat16().contiguous(memory_format=torch.channels_last)


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


def _layout(sizes, dtype=torch.float32):
    """One flat buffer of ``dtype`` (fp32 or bf16) holding the views of ``sizes`` in order: every view starts 16-byte
    aligned, and every element around them - at least GUARD before the first, directly after each view up to the next
    aligned start (at least GUARD) and after the last - is a guard word. Returns (views, buffer, guard slices)."""
    bits = {torch.float32: (torch.int32, GUARD_BITS), torch.bfloat16: (torch.int16, GUARD_BITS16)}
    itype, gbits = bits[dtype]
    align = 16 // torch.tensor([], dtype=dtype).element_size()
    starts, off = [], GUARD
    for s in sizes:
        starts.append(off)
        off = (off + s + GUARD + align - 1) // align * align
    buf = torch.full((off,), gbits, device=DEV, dtype=itype).view(dtype)
    views = [buf[a:a + s] for a, s in zip(starts, sizes)]
    ends = [0] + [a + s for a, s in zip(starts, sizes)]
    guards = [slice(e, a) for e, a in zip(ends, starts + [off])]
    return views, buf, guards


def _assert_guards(buf, guards, what):
    if buf.dtype == torch.bfloat16:
        b, gbits = buf.view(torch.int16), GUARD_BITS16
    else:
        b, gbits = _bits(buf), GUARD_BITS
    for g in guards:
        assert bool((b[g] == gbits).all()), f"{what}: guard elements {g.start}..{g.stop} overwritten"


def _prior(n, gen):
    """fp32 gradient already in the bucket: magnitudes up to ~1e3 (the addition rounds), every 7th value -0.0."""
    p = torch.randn(n, device=DEV, generator=gen) * torch.pow(10.0, torch.rand(n, device=DEV, generator=gen) * 5 - 2)
    p[::7] = -0.0
    return p


def _workspace(ws_bytes):
    if ws_bytes <= 0:
        return None
    return torch.full(((ws_bytes + 3) // 4,), float("nan"), device=DEV)


def _assert_bits_equal(got, want, what):
    g, w = _bits(got), _bits(want)
    bad = g != w
    if bool(bad.any()):
        i = int(bad.reshape(-1).nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ; first at {i}: got "
                             f"{float(got.reshape(-1)[i]):.9g}, want {float(want.reshape(-1)[i]):.9g}")


# ---------------------------------------------------------------------------------------------------------------------
# a. accumulating weight gradients
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(O.WGRAD_ACC_CASES))
def test_wgrad_acc_matches_prior_plus_overwrite(name):
    case = O.WGRAD_ACC_CASES[name]
    (n, h, w, cin, cout, k, stride, pad), ctas, _, path = case
    route, ws_bytes = O.case_route(case, _sms())
    assert route.path == path, route
    L = lib()
    full = L.hb_conv2d_wgrad_workspace_bytes(n, h, w, cin, cout, k, k, stride, pad, 1, ctas)
    assert full == route.ws_bytes, (full, route)
    gen = torch.Generator(device=DEV).manual_seed(len(name) * 31 + ctas)
    ho, wo = O.window_out(h, k, stride, pad), O.window_out(w, k, stride, pad)
    x, dy = _nhwc_bf16(n, cin, h, w, gen), _nhwc_bf16(n, cout, ho, wo, gen)
    m = cout * k * k * cin
    (dw,), buf, guards = _layout([m])
    prior = _prior(m, gen)
    dw.copy_(prior)
    ws = _workspace(ws_bytes)
    before = L.hb_launch_count()
    rc = L.hb_conv2d_wgrad_acc_bf16(ptr(x), ptr(dy), ptr(dw), ptr(ws), ws_bytes, n, h, w, cin, cout, k, k, stride, pad, 1,
                                    ctas, stream_ptr())
    torch.cuda.synchronize()
    _assert_guards(buf, guards, name)
    if path == O.REFUSED:
        assert rc == O.NOT_SUPPORTED, rc
        assert L.hb_launch_count() == before, "a refused call launched a kernel"
        _assert_bits_equal(dw, prior, name + ": refused call changed dw")
        return
    assert rc == 0, rc
    (over,), obuf, oguards = _layout([m])
    over.fill_(float("nan"))
    ws = _workspace(ws_bytes)
    assert L.hb_conv2d_wgrad_bf16(ptr(x), ptr(dy), ptr(over), ptr(ws), ws_bytes, n, h, w, cin, cout, k, k, stride, pad, 1,
                                  ctas, stream_ptr()) == 0
    torch.cuda.synchronize()
    _assert_guards(obuf, oguards, name + " overwrite")
    ref, abs_sum = wgrad_ref(x.float(), dy.float(), k, stride, pad)
    assert_within(over.view(cout, k, k, cin).cpu(), ref.permute(0, 2, 3, 1), abs_sum.permute(0, 2, 3, 1),
                  name + " overwrite", bits=FP32_BITS)
    _assert_bits_equal(dw, prior + over, name + ": accumulate != prior + overwrite")


@pytest.mark.parametrize("name", list(O.REPVGG_ACC_CASES))
def test_repvgg_wgrad_acc_matches_prior_plus_overwrite(name):
    case = O.REPVGG_ACC_CASES[name]
    (n, h, w, cin, cout), ctas, _, path = case
    route, ws_bytes = O.repvgg_case_route(case, _sms())
    assert route.path == path, route
    L = lib()
    assert L.hb_repvgg_wgrad_workspace_bytes(n, h, w, cin, cout, ctas) == route.ws_bytes
    gen = torch.Generator(device=DEV).manual_seed(len(name) * 17 + ctas)
    x, dy3, dy1 = _nhwc_bf16(n, cin, h, w, gen), _nhwc_bf16(n, cout, h, w, gen), _nhwc_bf16(n, cout, h, w, gen)
    m3, m1 = cout * 9 * cin, cout * cin
    # the bucket's order: the 1x1 branch (registered after the 3x3 one) lies BEFORE it
    (dw1, dw3), buf, guards = _layout([m1, m3])
    p1, p3 = _prior(m1, gen), _prior(m3, gen)
    dw1.copy_(p1)
    dw3.copy_(p3)
    ws = _workspace(ws_bytes)
    before = L.hb_launch_count()
    rc = L.hb_repvgg_wgrad_acc_bf16(ptr(x), ptr(dy3), ptr(dy1), ptr(dw3), ptr(dw1), ptr(ws), ws_bytes, n, h, w, cin, cout,
                                    ctas, stream_ptr())
    torch.cuda.synchronize()
    _assert_guards(buf, guards, name)
    if path == O.REFUSED:
        assert rc == O.NOT_SUPPORTED, rc
        assert L.hb_launch_count() == before, "a refused call launched a kernel"
        _assert_bits_equal(dw3, p3, name + ": refused call changed dW3")
        _assert_bits_equal(dw1, p1, name + ": refused call changed dW1")
        return
    assert rc == 0, rc
    (over,), obuf, oguards = _layout([m3 + m1])
    over.fill_(float("nan"))
    ws = _workspace(ws_bytes)
    assert L.hb_repvgg_wgrad_bf16(ptr(x), ptr(dy3), ptr(dy1), ptr(over), ptr(ws), ws_bytes, n, h, w, cin, cout, ctas,
                                  stream_ptr()) == 0
    torch.cuda.synchronize()
    _assert_guards(obuf, oguards, name + " overwrite")
    r3, a3 = wgrad_ref(x.float(), dy3.float(), 3, 1, 1)
    r1, a1 = wgrad_ref(x.float(), dy1.float(), 1)
    assert_within(over[:m3].view(cout, 3, 3, cin).cpu(), r3.permute(0, 2, 3, 1), a3.permute(0, 2, 3, 1),
                  name + " overwrite dW3", bits=FP32_BITS)
    assert_within(over[m3:].view(cout, 1, 1, cin).cpu(), r1.permute(0, 2, 3, 1), a1.permute(0, 2, 3, 1),
                  name + " overwrite dW1", bits=FP32_BITS)
    _assert_bits_equal(dw3, p3 + over[:m3], name + ": dW3 accumulate != prior + overwrite")
    _assert_bits_equal(dw1, p1 + over[m3:], name + ": dW1 accumulate != prior + overwrite")


# ---------------------------------------------------------------------------------------------------------------------
# b. filter packing
# ---------------------------------------------------------------------------------------------------------------------
# name -> (Cout, Cin, R, S, CinP, CinD, CoutP, CoutF, with wd); packed sizes around the 4096-element chunks
PACK_CASES = {
    "nf4095-nowd": (13, 35, 3, 3, 35, 0, 0, 13, False),
    "nf4097-nowd-cinp": (17, 240, 1, 1, 241, 0, 0, 17, False),
    "nf8191-nowd-cinp": (1, 8190, 1, 1, 8191, 0, 0, 1, False),
    "nf8193-nowd-coutf": (2, 2730, 1, 1, 2731, 0, 0, 3, False),
    "nf1-nd8192-padded": (1, 1, 1, 1, 1, 128, 64, 1, True),
    "nf4000-nd8192-4x4": (10, 25, 4, 4, 25, 32, 16, 10, True),
    "padded-3x3": (24, 20, 3, 3, 24, 32, 32, 32, True),
    "exact-3x3": (32, 16, 3, 3, 16, 16, 32, 32, True),
    "tiny-1x1": (8, 8, 1, 1, 8, 16, 16, 16, True),
}


def _pack_outputs(cout, cin, r, s, cinp, cind, coutp, coutf, with_wd):
    nf, nd = coutf * r * s * cinp, (cind * r * s * coutp if with_wd else 0)
    views, buf, guards = _layout([nf] + ([nd] if with_wd else []), torch.bfloat16)
    for v in views:
        v.fill_(float("nan"))
    return views[0], (views[1] if with_wd else None), buf, guards


def _check_pack(wf, wd, w, case, what):
    cout, cin, r, s, cinp, cind, coutp, coutf, with_wd = case
    ok, nbad = O.bf16_equal(wf, O.pack_wf(w, coutf, cinp))
    assert ok, f"{what}: {nbad} wf elements differ from the restatement"
    if with_wd:
        ok, nbad = O.bf16_equal(wd, O.pack_wd(w, cind, coutp))
        assert ok, f"{what}: {nbad} wd elements differ from the restatement"


def _masters(case, seed):
    cout, cin, r, s = case[:4]
    return O.masters((cout, r, s, cin), torch.Generator().manual_seed(seed)).to(DEV)


@pytest.mark.parametrize("name", list(PACK_CASES))
def test_pack_single_matches_restatement(name):
    case = PACK_CASES[name]
    w = _masters(case, len(name))
    wf, wd, buf, guards = _pack_outputs(*case)
    cout, cin, r, s, cinp, cind, coutp, coutf, _ = case
    assert lib().hb_pack_conv_weights(ptr(w), ptr(wf), ptr(wd), cout, cin, r, s, cinp, cind, coutp, coutf,
                                      stream_ptr()) == 0
    torch.cuda.synchronize()
    _assert_guards(buf, guards, name)
    _check_pack(wf, wd, w, case, name)


def test_pack_multi_matches_restatement():
    """Every PACK_CASES filter in one table (with and without wd), one launch; chunk k of a filter covers packed elements
    [4096 k, 4096 k + 4096) of wf followed by wd."""
    L = lib()
    chunk = L.hb_pack_chunk_elems()
    assert chunk == 4096
    dt = np.dtype([("ptrs", "<u8", (3,)), ("ints", "<i4", (8,))])
    assert dt.itemsize == L.hb_pack_meta_bytes()
    cases = list(PACK_CASES.items())
    metas = np.zeros(len(cases), dtype=dt)
    rows, keep = [], []
    for i, (name, case) in enumerate(cases):
        cout, cin, r, s, cinp, cind, coutp, coutf, with_wd = case
        w = _masters(case, 100 + i)
        wf, wd, buf, guards = _pack_outputs(*case)
        keep.append((name, case, w, wf, wd, buf, guards))
        metas[i]["ptrs"] = (w.data_ptr(), wf.data_ptr(), 0 if wd is None else wd.data_ptr())
        metas[i]["ints"] = (cout, cin, r, s, cinp, cind, coutp, coutf)
        total = wf.numel() + (0 if wd is None else wd.numel())
        nch = (total + chunk - 1) // chunk
        rows.append(np.stack([np.full(nch, i, dtype=np.int32), np.arange(nch, dtype=np.int32)], 1))
    chunks = np.ascontiguousarray(np.concatenate(rows, 0))
    md = torch.from_numpy(metas.view(np.uint8).reshape(len(cases), -1).copy()).to(DEV)
    cd = torch.from_numpy(chunks).to(DEV)
    assert L.hb_pack_conv_weights_multi(ptr(md), ptr(cd), int(chunks.shape[0]), stream_ptr()) == 0
    torch.cuda.synchronize()
    for name, case, w, wf, wd, buf, guards in keep:
        _assert_guards(buf, guards, "multi " + name)
        _check_pack(wf, wd, w, case, "multi " + name)


@pytest.mark.parametrize("cout,cin,cind,coutp", [(16, 16, 16, 16), (24, 20, 32, 32), (3, 5, 16, 16), (48, 96, 96, 48)])
def test_pack_dgrad_s2_matches_restatement(cout, cin, cind, coutp):
    w = O.masters((cout, 3, 3, cin), torch.Generator().manual_seed(cout * cin)).to(DEV)
    n = 9 * cind * coutp
    (out,), buf, guards = _layout([n], torch.bfloat16)
    out.fill_(float("nan"))
    assert lib().hb_pack_dgrad_s2_weights(ptr(w), ptr(out), cout, cin, cind, coutp, stream_ptr()) == 0
    torch.cuda.synchronize()
    _assert_guards(buf, guards, "dgrad_s2")
    ok, nbad = O.bf16_equal(out, O.pack_dgrad_s2(w, cind, coutp))
    assert ok, f"{nbad} class-filter elements differ from the restatement"


def _check_pack_cache_entry(wt, master, what):
    ent = _fused._pack_cache[id(wt)]
    m = master.detach().permute(0, 2, 3, 1)
    ok, nbad = O.bf16_equal(ent.wf, O.pack_wf(m, ent.cout_p, ent.cin_p))
    assert ok, f"{what}: {nbad} wf elements do not match the current master"
    if ent.wd is not None:
        ok, nbad = O.bf16_equal(ent.wd, O.pack_wd(m, ent.cin_d, ent.cout_p))
        assert ok, f"{what}: {nbad} wd elements do not match the current master"


def test_pack_table_repacks_every_filter_after_an_update():
    """Three channels_last filters join the table; after an in-place update of all three, ONE forward through the first
    re-packs every registered filter (one multi-tensor launch): each cache entry matches its new master."""
    gc.collect()
    gen = torch.Generator().manual_seed(5)
    shapes = [(32, 16, 3, 3), (48, 24, 1, 1), (24, 20, 3, 3)]      # the last: Cout and Cin padded
    ws = [torch.nn.Parameter(torch.randn(s, generator=gen).to(DEV).contiguous(memory_format=torch.channels_last))
          for s in shapes]
    xs = [torch.randn(2, s[1], 10, 10, device=DEV).requires_grad_(i != 1) for i, s in enumerate(shapes)]
    for x, wt in zip(xs, ws):
        _fused.conv2d(x, wt, None, 1, wt.shape[2] // 2)
    for i, wt in enumerate(ws):
        new = O.masters(wt.shape, torch.Generator().manual_seed(50 + i), edges=True)
        # the edge values go to a KRSC prefix: the packed filters see them in channel order
        with torch.no_grad():
            wt.copy_(new.view(wt.shape[0], wt.shape[2], wt.shape[3], wt.shape[1]).permute(0, 3, 1, 2).to(DEV))
        torch.autograd.graph.increment_version([wt])
    L = lib()
    before = L.hb_launch_count()
    _fused.conv2d(xs[0], ws[0], None, 1, 1)
    torch.cuda.synchronize()
    assert L.hb_launch_count() - before == 2, "expected one packing launch and one convolution"
    for i, wt in enumerate(ws):
        _check_pack_cache_entry(wt, wt, f"filter {i}")


# ---------------------------------------------------------------------------------------------------------------------
# c. gradient clipping
# ---------------------------------------------------------------------------------------------------------------------
def _clip(g, max_norm):
    """Runs hb_grad_clip_norm on a guarded copy of g: (result, reported norm, guard ok)."""
    n = g.numel()
    (v,), buf, guards = _layout([n])
    v.copy_(g)
    L = lib()
    scratch = torch.full((L.hb_grad_clip_partials_max(),), float("nan"), device=DEV, dtype=torch.float64)
    ctl = torch.zeros(8, device=DEV)
    assert L.hb_grad_clip_norm(ptr(v), n, ctypes.c_float(max_norm), ptr(scratch), ptr(ctl), stream_ptr()) == 0
    torch.cuda.synchronize()
    _assert_guards(buf, guards, f"clip n={n}")
    return v.clone(), float(ctl[7])


def _clip_sizes():
    big = _sms() * 4 * 1024 * 2 + 7          # past grid x 1024: the grid-stride loops wrap
    return [1, 3, 4, 5, 4097, 4098, 4099, big]


def _assert_clip_equal(got, want, what):
    g, w = got.cpu(), want.cpu()
    same = (_bits(g) == _bits(w)) | (torch.isnan(g) & torch.isnan(w))
    assert bool(same.all()), f"{what}: {int((~same).sum())} of {same.numel()} elements differ from fl32(g * coef)"


@pytest.mark.parametrize("kind", ["active", "below", "inf", "nan"])
def test_grad_clip_per_element(kind):
    for n in _clip_sizes():
        gen = torch.Generator(device=DEV).manual_seed(n)
        g = torch.randn(n, device=DEV, generator=gen) * 3
        g[1::5] = -0.0
        if kind == "inf":
            g[n // 2] = float("inf")
        if kind == "nan":
            g[n - 1] = float("nan")
        norm64 = O.norm_ref(g)
        max_norm = {"active": 0.25 * norm64, "below": 2.0 * norm64 + 1.0}.get(kind, 1.0)
        max_norm = float(torch.tensor(max_norm, dtype=torch.float32))
        out, norm_k = _clip(g, max_norm)
        what = f"{kind} n={n}"
        if kind in ("active", "below"):
            ulp = float(torch.tensor(norm64, dtype=torch.float32).nextafter(torch.tensor(float("inf"))) -
                        torch.tensor(norm64, dtype=torch.float32))
            assert abs(norm_k - norm64) <= ulp, f"{what}: norm {norm_k!r} vs fp64 {norm64!r}"
        if kind == "below":
            _assert_bits_equal(out, g, what + ": below the threshold the buffer changed")
            continue
        if kind == "inf":
            assert norm_k == float("inf")
        if kind == "nan":
            assert norm_k != norm_k
            assert bool(torch.isnan(out).all()), f"{what}: a NaN norm must make every gradient NaN"
        _assert_clip_equal(out, O.clip_ref(g, norm_k, max_norm), what)


def test_grad_clip_refusals():
    L = lib()
    scratch = torch.empty(L.hb_grad_clip_partials_max(), device=DEV, dtype=torch.float64)
    buf = torch.randn(64, device=DEV)
    keep = buf.clone()
    c = ctypes.c_float(0.1)
    assert L.hb_grad_clip_norm(ctypes.c_void_p(buf.data_ptr() + 4), 60, c, ptr(scratch), None, stream_ptr()) == MISALIGNED
    assert L.hb_grad_clip_norm(ptr(buf), 0, c, ptr(scratch), None, stream_ptr()) == INVALID
    assert L.hb_grad_clip_norm(ptr(buf), -4, c, ptr(scratch), None, stream_ptr()) == INVALID
    assert L.hb_grad_clip_norm(ptr(buf), 64, c, None, None, stream_ptr()) == INVALID
    torch.cuda.synchronize()
    _assert_bits_equal(buf, keep, "a refused clip changed the buffer")


# ---------------------------------------------------------------------------------------------------------------------
# d. direct bucket accumulation == autograd accumulation, by route
# ---------------------------------------------------------------------------------------------------------------------
R_REPVGG, R_ACC, R_801, R_PADDED, R_STEM, R_BN = O.R_REPVGG, O.R_ACC, O.R_801, O.R_PADDED, O.R_STEM, O.R_BN
_WATCH = ("hb_repvgg_wgrad_acc_bf16", "hb_conv2d_wgrad_acc_bf16", "hb_conv2d_wgrad_bf16", "hb_repvgg_wgrad_bf16",
          "hb_im2col_smallc_bf16", "hb_bn_act_bwd_bf16")


class _Recorder:
    """Stands in for the library handle of nn/_fused.py and records the calls that decide a gradient's route."""

    def __init__(self, real):
        self.real, self.calls = real, []

    def __getattr__(self, name):
        fn = getattr(self.real, name)
        if name not in _WATCH:
            return fn

        def wrapped(*args):
            rc = fn(*args)
            self.calls.append((name, args, rc))
            return rc
        return wrapped

    def routes(self):
        out, stem_seen = set(), False
        for i, (name, args, rc) in enumerate(self.calls):
            if name == "hb_im2col_smallc_bf16":
                stem_seen = True
            elif name == "hb_repvgg_wgrad_acc_bf16" and rc == 0:
                out.add(R_REPVGG)
            elif name == "hb_conv2d_wgrad_acc_bf16":
                out.add(R_ACC if rc == 0 else R_801 if rc == O.NOT_SUPPORTED else f"error {rc}")
            elif name == "hb_conv2d_wgrad_bf16":
                prev = self.calls[i - 1] if i else None
                if prev and prev[0] == "hb_conv2d_wgrad_acc_bf16" and prev[2] == O.NOT_SUPPORTED:
                    continue                                   # the refusal's overwriting fall-back
                # the stem's gradient: a 1x1 weight gradient over its 32 im2col columns
                out.add(R_STEM if stem_seen and args[10] == 1 and args[8] == 32 else R_PADDED)
            elif name == "hb_repvgg_wgrad_bf16":
                out.add(R_PADDED)                              # a direct bucket only refuses it for padded channels
            elif name == "hb_bn_act_bwd_bf16" and args[17] is not None:
                out.add(R_BN)
        return out

    def planned(self):
        """(route, (kind, shape)) of every accumulating weight-gradient call, as _grad_bucket_oracle.DIRECT_WITNESSES
        writes them."""
        out = set()
        for name, args, rc in self.calls:
            if name == "hb_repvgg_wgrad_acc_bf16":
                out.add((R_REPVGG if rc == 0 else f"rc {rc}", ("repvgg", tuple(args[7:12]))))
            elif name == "hb_conv2d_wgrad_acc_bf16":
                out.add((R_ACC if rc == 0 else R_801 if rc == O.NOT_SUPPORTED else f"rc {rc}",
                         ("wgrad", tuple(args[5:11]) + tuple(args[12:14]))))
        return out


def _block(cin, cout, stride, identity):
    def make():
        return RepBlock(cin, cout, stride, identity)
    return make


def _model(factory):
    def make():
        return getattr(hb.models, factory)(num_classes=10)
    return make


# name -> (factory, input shape, input needs grad); the routes each case takes are _grad_bucket_oracle.DIRECT_ROUTES
DIRECT_CASES = {
    "repblock-s1-identity": (_block(48, 48, 1, True), (4, 48, 16, 16), True),
    "repblock-s1": (_block(32, 64, 1, False), (2, 32, 24, 20), True),
    "repblock-s2": (_block(48, 64, 2, False), (4, 48, 32, 32), True),
    "repblock-s2-single-range": (_block(128, 256, 2, False), (2, 128, 4, 4), True),
    "repblock-s1-padded": (_block(12, 32, 1, False), (2, 12, 16, 16), True),
    "repblock-stem": (_block(3, 48, 2, False), (2, 3, 32, 32), False),
    "repvgg_a0": (_model("repvgg_a0"), (4, 3, 64, 64), False),
    "rexnet1_0x": (_model("rexnet1_0x"), (4, 3, 64, 64), False),
    "resnet18": (_model("resnet18"), (4, 3, 64, 64), True),
}


def test_direct_cases_reach_all_six_routes():
    assert set(DIRECT_CASES) == set(O.DIRECT_ROUTES)
    assert set().union(*O.DIRECT_ROUTES.values()) == O.ALL_ROUTES


def _direct_ids():
    return [f"{k}-" + "+".join(sorted(O.DIRECT_ROUTES[k])) for k in DIRECT_CASES]


@pytest.mark.parametrize("name", list(DIRECT_CASES), ids=_direct_ids())
def test_direct_grads_match_autograd_accumulation(name, monkeypatch):
    factory, shape, x_grad = DIRECT_CASES[name]
    routes = O.DIRECT_ROUTES[name]
    gen = torch.Generator().manual_seed(3)
    xs = [torch.randn(shape, generator=gen).to(DEV) for _ in range(2)]
    blocks = factory().__class__ is RepBlock
    if blocks:
        ups = [torch.randn(1, generator=gen).item() + torch.randn(shape[0], 1, 1, 1, generator=gen).to(DEV)
               for _ in range(2)]
    ts = [torch.randint(0, 10, (shape[0],), generator=gen).to(DEV) for _ in range(2)]
    arms = {}
    for direct in (True, False):
        torch.manual_seed(0)
        m = factory().to(DEV).to(memory_format=torch.channels_last).train()
        bucket = GradBucket(m.parameters(), direct=direct)
        rec = _Recorder(_fused.lib())
        monkeypatch.setattr(_fused, "lib", lambda rec=rec: rec)
        dxs = []
        for i in range(2):
            x = xs[i].clone().requires_grad_(x_grad)
            y = m(x)
            loss = (y.float() * ups[i]).sum() if blocks else TF.cross_entropy(y, ts[i], label_smoothing=0.1)
            loss.backward()
            if x_grad:
                dxs.append(x.grad)
        torch.cuda.synchronize()
        monkeypatch.undo()
        arms[direct] = (m, bucket, dxs, rec)
    (md, bd, dxd, rec), (ma, ba, dxa, _) = arms[True], arms[False]
    for (n, pd), pa in zip(md.named_parameters(), ma.parameters()):
        _assert_bits_equal(pd.grad, pa.grad, f"{name}: .grad of {n}")
    _assert_bits_equal(bd.flat, ba.flat, f"{name}: bucket")
    for i, (a, b) in enumerate(zip(dxd, dxa)):
        _assert_bits_equal(a, b, f"{name}: input gradient of micro-batch {i}")
    assert rec.routes() == routes, f"routes taken: {sorted(rec.routes())}"
    # the calls the CPU test holds to their routes for every SM count are made here, and take those routes
    missing = [w for w in O.DIRECT_WITNESSES[name] if w not in rec.planned()]
    assert not missing, f"witness calls not made: {missing}; made: {sorted(rec.planned())}"


# ---------------------------------------------------------------------------------------------------------------------
# e. graph replay == eager
# ---------------------------------------------------------------------------------------------------------------------
def _train_arm(factory):
    torch.manual_seed(0)
    m = getattr(hb.models, factory)(num_classes=10).to(DEV).to(memory_format=torch.channels_last).train()
    bucket = GradBucket(m.parameters())
    opt = hb.optim.AdaBelief(m.parameters(), lr=1e-3, betas=(0.95, 0.99), eps=1e-6, capturable=True)

    def step(x, t):
        loss = TF.cross_entropy(m(x), t, label_smoothing=0.1)
        loss.backward()
        opt.step()
        bucket.zero_()
        return loss
    return m, opt, step


def _state_tensors(m, opt):
    out = [(f"param {n}", p) for n, p in m.named_parameters()]
    out += [(f"buffer {n}", b) for n, b in m.named_buffers()]
    for i, p in enumerate(m.parameters()):
        for k, v in opt.state[p].items():
            if torch.is_tensor(v):
                out.append((f"optimizer state {k} of parameter {i}", v))
    return out


def _snapshot(m, opt):
    return [(n, t.detach().clone()) for n, t in _state_tensors(m, opt)]


def _assert_same_state(got, want, what):
    assert len(got) == len(want) and len(got) > 0
    for (n, x), (_, y) in zip(got, want):
        if x.dtype.is_floating_point:
            _assert_bits_equal(x.float(), y.float(), f"{what}: {n}")
        else:
            assert torch.equal(x, y), f"{what}: {n}"


SEED_WARMUP = 7


def _seed_step(i):
    """Both arms draw ReXNet's head-dropout mask from the global CUDA generator: reseeding it before every eager step and
    every replay gives both the same mask (a replay starts from the generator's current seed and offset)."""
    torch.cuda.manual_seed(1000 + i)


@pytest.mark.parametrize("factory", ["repvgg_a0", "rexnet1_0x", "resnet18"])
def test_graph_replay_matches_eager_bit_for_bit(factory):
    """The eager arm runs its whole history first and is kept alive, so no eager forward re-packs the graphed model's
    filters: after each replay, the packed filters of the graphed model can only have come from the graph's own repack."""
    gc.collect()            # no dead filter may leave the packing table while the graph holds it
    gen = torch.Generator().manual_seed(11)
    xs = [torch.randn(8, 3, 64, 64, generator=gen).to(DEV) for _ in range(3)]
    ts = [torch.randint(0, 10, (8,), generator=gen).to(DEV) for _ in range(3)]
    me, oe, step_e = _train_arm(factory)
    torch.cuda.manual_seed(SEED_WARMUP)
    for _ in range(2):
        step_e(xs[0], ts[0])
    snaps, losses = [_snapshot(me, oe)], []
    for i, (x, t) in enumerate(zip(xs, ts)):
        _seed_step(i)
        losses.append(step_e(x, t).detach().clone())
        snaps.append(_snapshot(me, oe))
    torch.cuda.synchronize()

    mg, og, step_g = _train_arm(factory)
    torch.cuda.manual_seed(SEED_WARMUP)
    graphed = GraphedTrainStep(step_g, (xs[0], ts[0]), warmup=2)
    assert graphed.launches_per_replay > 50
    torch.cuda.synchronize()
    _assert_same_state(_snapshot(mg, og), snaps[0], "after the warm-ups")
    for i, (x, t) in enumerate(zip(xs, ts)):
        masters = {id(p): p.detach().clone() for p in mg.parameters()}
        _seed_step(i)
        lg = graphed(x, t)
        torch.cuda.synchronize()
        # this replay packed every filter of the graphed model from the masters it started with
        n = 0
        for p in mg.parameters():
            ent = _fused._pack_cache.get(id(p))
            if ent is not None and ent.wref() is p:
                _check_pack_cache_entry(p, masters[id(p)], f"{factory} step {i}: packed {tuple(p.shape)} filter")
                n += 1
        assert n > 0
        _assert_bits_equal(lg, losses[i], f"loss of step {i}")
        _assert_same_state(_snapshot(mg, og), snaps[i + 1], f"step {i}")
