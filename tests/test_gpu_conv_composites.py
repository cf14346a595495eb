"""GPU parity tests, through the C ABI, for the composite convolution entry points of a RepVGG block's backward pass:

  hb_conv3x3_accum_bf16      dX = dgrad3x3(dY3) + dgrad1x1(dY1) + dX_identity in one accumulator
  hb_conv2d_dgrad_s2_bf16    stride-2 data gradient by output-parity classes (+ the 1x1 stride-2 branch)
  hb_repvgg_wgrad_bf16       dW3 and dW1 in one pass over x (row-window kernel, deterministic reduction)
  hb_pack_conv_weights_multi all filters of a network packed by one launch

Reference: torch fp32 autograd on the CPU on the same bf16-rounded operands (reference semantics:
holocron/models/classification/repvgg.py:55-73 = nn.Conv2d 3x3 p1 + nn.Conv2d 1x1 + identity, summed).
Tolerances: bf16 outputs rel-L2 < 4e-3; fp32 weight gradients < 1e-3 (north_star); deterministic kernels bit-equal
between two runs. Every element also lies within the per-element bound of tests/_bounds.py (fp64 on the same operands)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as TF

from holocron_b200._lib import lib, ptr, stream_ptr

from _bounds import FP32_BITS, assert_within, dgrad_ref, ulp, wgrad_ref

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous().cuda()


@pytest.mark.parametrize("case", [(2, 14, 14, 48, 2), (2, 56, 56, 48, 1), (3, 112, 112, 48, 2), (2, 28, 28, 64, 0),
                                  (2, 30, 20, 32, 2), (2, 9, 11, 16, 1)])
def test_accumulated_block_dgrad(case):
    n, h, w, c, nextra = case
    torch.manual_seed(0)
    L = lib()
    dy3, dy1, dxid = (torch.randn(n, c, h, w).bfloat16() for _ in range(3))
    w3 = (torch.randn(c, c, 3, 3) / (9 * c) ** 0.5).bfloat16().float()
    w1 = (torch.randn(c, c, 1, 1) / c ** 0.5).bfloat16().float()
    # reference: gradient of  sum(conv3x3(x) * dy3) + sum(conv1x1(x) * dy1) + sum(x * dxid)  w.r.t. x
    x = torch.zeros(n, c, h, w, requires_grad=True)
    tot = (TF.conv2d(x, w3, padding=1) * dy3.float()).sum()
    if nextra >= 1:
        tot = tot + (TF.conv2d(x, w1) * dy1.float()).sum()
    if nextra >= 2:
        tot = tot + (x * dxid.float()).sum()
    (ref,) = torch.autograd.grad(tot, x)
    wf = torch.empty(c, 3, 3, c, device="cuda", dtype=torch.bfloat16)
    wd3 = torch.empty(c, 3, 3, c, device="cuda", dtype=torch.bfloat16)
    assert L.hb_pack_conv_weights(ptr(w3.permute(0, 2, 3, 1).contiguous().cuda()), ptr(wf), ptr(wd3), c, c, 3, 3, c, c, c, c,
                                  stream_ptr()) == 0
    wf1 = torch.empty(c, 1, 1, c, device="cuda", dtype=torch.bfloat16)
    wd1 = torch.empty(c, 1, 1, c, device="cuda", dtype=torch.bfloat16)
    assert L.hb_pack_conv_weights(ptr(w1.permute(0, 2, 3, 1).contiguous().cuda()), ptr(wf1), ptr(wd1), c, c, 1, 1, c, c, c, c,
                                  stream_ptr()) == 0
    eye = torch.eye(c, device="cuda", dtype=torch.bfloat16).reshape(c, 1, 1, c).contiguous()
    d3, d1, di = nhwc(dy3), nhwc(dy1), nhwc(dxid)
    out = torch.full((n, h, w, c), float("nan"), device="cuda", dtype=torch.bfloat16)
    rc = L.hb_conv3x3_accum_bf16(ptr(d3), ptr(wd3), ptr(d1) if nextra >= 1 else ptr(None), ptr(wd1) if nextra >= 1 else ptr(None),
                                 ptr(di) if nextra >= 2 else ptr(None), ptr(eye) if nextra >= 2 else ptr(None), nextra, ptr(out),
                                 n, h, w, c, c, 0, stream_ptr())
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert rel_l2(out, ref.permute(0, 2, 3, 1)) < 4e-3
    r, a = dgrad_ref(x.shape, w3, dy3, 1, 1)
    if nextra >= 1:
        r1, a1 = dgrad_ref(x.shape, w1, dy1)
        r, a = r + r1, a + a1
    if nextra >= 2:
        r, a = r + dxid.double(), a + dxid.double().abs()
    assert_within(out.permute(0, 3, 1, 2), r, a, "dX")


def test_accum_reports_unsupported_shapes():
    """Shapes outside the shared-memory-resident scheme return cudaErrorNotSupported (801) without launching."""
    L = lib()
    t = torch.zeros(1, 8, 8, 256, device="cuda", dtype=torch.bfloat16)
    wz = torch.zeros(256, 3, 3, 256, device="cuda", dtype=torch.bfloat16)
    before = L.hb_launch_count()
    assert L.hb_conv3x3_accum_bf16(ptr(t), ptr(wz), ptr(None), ptr(None), ptr(None), ptr(None), 0, ptr(t.clone()), 1, 8, 8, 256,
                                   256, 0, stream_ptr()) == 801
    assert L.hb_launch_count() == before
    assert L.hb_repvgg_wgrad_workspace_bytes(2, 7, 7, 1280, 1280, 0) == 0


@pytest.mark.parametrize("case", [(2, 16, 16, 48, 48, True), (2, 16, 16, 48, 96, False), (3, 15, 9, 24, 32, True),
                                  (2, 14, 14, 192, 1280, True), (2, 7, 7, 64, 64, False), (4, 56, 56, 48, 96, True),
                                  (1, 2, 2, 16, 16, True), (2, 224, 224, 8, 48, False)])
def test_parity_class_stride2_dgrad(case):
    n, h, w, cin, cout, with1x1 = case
    torch.manual_seed(4)
    L = lib()
    w3 = (torch.randn(cout, cin, 3, 3) / (cin * 9) ** 0.5).bfloat16().float()
    w1 = (torch.randn(cout, cin, 1, 1) / cin ** 0.5).bfloat16().float()
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    dy3, dy1 = torch.randn(n, cout, ho, wo).bfloat16(), torch.randn(n, cout, ho, wo).bfloat16()
    x = torch.zeros(n, cin, h, w, requires_grad=True)
    tot = (TF.conv2d(x, w3, stride=2, padding=1) * dy3.float()).sum()
    if with1x1:
        tot = tot + (TF.conv2d(x, w1, stride=2) * dy1.float()).sum()
    (ref,) = torch.autograd.grad(tot, x)
    cind = (cin + 15) // 16 * 16
    wcls = torch.empty(9 * cind * cout, device="cuda", dtype=torch.bfloat16)
    assert L.hb_pack_dgrad_s2_weights(ptr(w3.permute(0, 2, 3, 1).contiguous().cuda()), ptr(wcls), cout, cin, cind, cout,
                                      stream_ptr()) == 0
    wd1 = torch.zeros(cind, 1, 1, cout, device="cuda", dtype=torch.bfloat16)
    wd1[:cin, 0, 0, :] = w1[:, :, 0, 0].t().cuda().bfloat16()
    d3, d1 = nhwc(dy3), nhwc(dy1)
    dx = torch.full((n, h, w, cind), float("nan"), device="cuda", dtype=torch.bfloat16)
    rc = L.hb_conv2d_dgrad_s2_bf16(ptr(d3), ptr(wcls), ptr(d1) if with1x1 else ptr(None), ptr(wd1) if with1x1 else ptr(None),
                                   ptr(dx), n, h, w, ho, wo, cout, cind, 0, stream_ptr())
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert rel_l2(dx[..., :cin], ref.permute(0, 2, 3, 1)) < 4e-3
    r, a = dgrad_ref((n, cin, h, w), w3, dy3, 2, 1)
    slack = None
    if with1x1:
        # the 1x1 branch is stored (bf16) first; class (0, 0) of the 3x3 part is rounded to bf16 and added onto it
        r1, a1 = dgrad_ref((n, cin, h, w), w1, dy1, 2, 0)
        slack = torch.zeros_like(r)
        slack[:, :, ::2, ::2] = 0.5 * (ulp(r) + ulp(r1))[:, :, ::2, ::2]
        r, a = r + r1, a + a1
    assert_within(dx[..., :cin].permute(0, 3, 1, 2), r, a, "dX", slack=slack)
    assert bool((dx[..., cin:] == 0).all())           # padded channels: written, exactly zero
    assert torch.isfinite(dx.float()).all()            # every element of dx is written by exactly one class


@pytest.mark.parametrize("case", [(3, 112, 112, 48, 48), (5, 28, 28, 96, 96), (40, 14, 14, 192, 192), (2, 30, 20, 32, 48),
                                  (2, 16, 16, 72, 200), (2, 9, 11, 16, 16), (300, 14, 14, 48, 48)])
def test_block_wgrad_one_pass(case):
    n, h, w, cin, cout = case
    torch.manual_seed(6)
    L = lib()
    x = torch.randn(n, cin, h, w).bfloat16()
    dy3, dy1 = torch.randn(n, cout, h, w).bfloat16(), torch.randn(n, cout, h, w).bfloat16()
    w3 = torch.zeros(cout, cin, 3, 3, requires_grad=True)
    w1 = torch.zeros(cout, cin, 1, 1, requires_grad=True)
    tot = (TF.conv2d(x.float(), w3, padding=1) * dy3.float()).sum() + (TF.conv2d(x.float(), w1) * dy1.float()).sum()
    g3, g1 = torch.autograd.grad(tot, (w3, w1))
    wsb = L.hb_repvgg_wgrad_workspace_bytes(n, h, w, cin, cout, 0)
    assert wsb > 0
    xn, d3, d1 = nhwc(x), nhwc(dy3), nhwc(dy1)
    outs = []
    for _ in range(2):
        ws = torch.empty(wsb // 4, device="cuda")
        dw = torch.full((cout * 10 * cin,), float("nan"), device="cuda")
        assert L.hb_repvgg_wgrad_bf16(ptr(xn), ptr(d3), ptr(d1), ptr(dw), ptr(ws), wsb, n, h, w, cin, cout, 0, stream_ptr()) == 0
        torch.cuda.synchronize()
        outs.append(dw)
    assert torch.equal(outs[0], outs[1])               # fixed-order reduction: bit-reproducible
    assert rel_l2(outs[0][:cout * 9 * cin].view(cout, 3, 3, cin), g3.permute(0, 2, 3, 1)) < 1e-3
    assert rel_l2(outs[0][cout * 9 * cin:].view(cout, 1, 1, cin), g1.permute(0, 2, 3, 1)) < 1e-3
    dw = outs[0].cpu()
    r3, a3 = wgrad_ref(x, dy3, 3, 1, 1)
    r1, a1 = wgrad_ref(x, dy1, 1)
    assert_within(dw[:cout * 9 * cin].view(cout, 3, 3, cin), r3.permute(0, 2, 3, 1), a3.permute(0, 2, 3, 1), "dW3",
                  bits=FP32_BITS)
    assert_within(dw[cout * 9 * cin:].view(cout, 1, 1, cin), r1.permute(0, 2, 3, 1), a1.permute(0, 2, 3, 1), "dW1",
                  bits=FP32_BITS)


def test_generic_wgrad_is_deterministic_with_workspace():
    torch.manual_seed(7)
    L = lib()
    n, h, w, cin, cout = 8, 7, 7, 1280, 1280          # generic split-K kernel (row-window scheme not eligible)
    x = torch.randn(n, h, w, cin, device="cuda").bfloat16()
    dy = torch.randn(n, h, w, cout, device="cuda").bfloat16()
    wsb = L.hb_conv2d_wgrad_workspace_bytes(n, h, w, cin, cout, 3, 3, 1, 1, 1, 0)
    outs = []
    for _ in range(2):
        ws = torch.empty(max(wsb // 4, 1), device="cuda")
        dw = torch.empty(cout, 3, 3, cin, device="cuda")
        assert L.hb_conv2d_wgrad_bf16(ptr(x), ptr(dy), ptr(dw), ptr(ws), wsb, n, h, w, cin, cout, 3, 3, 1, 1, 1, 0,
                                      stream_ptr()) == 0
        torch.cuda.synchronize()
        outs.append(dw)
    assert torch.equal(outs[0], outs[1])
    wt = torch.zeros(cout, cin, 3, 3, device="cuda", requires_grad=True)
    y = TF.conv2d(x.permute(0, 3, 1, 2).float(), wt, padding=1)
    (g,) = torch.autograd.grad(y, wt, dy.permute(0, 3, 1, 2).float())
    assert rel_l2(outs[0], g.permute(0, 2, 3, 1)) < 1e-3
    r, a = wgrad_ref(x.permute(0, 3, 1, 2), dy.permute(0, 3, 1, 2), 3, 1, 1)
    assert_within(outs[0].cpu(), r.permute(0, 2, 3, 1), a.permute(0, 2, 3, 1), "dW", bits=FP32_BITS)


def test_multi_tensor_filter_packing_matches_single():
    torch.manual_seed(8)
    L = lib()
    shapes = [(48, 3, 3, 3, 8), (48, 48, 3, 3, 48), (96, 48, 1, 1, 48), (1280, 192, 3, 3, 192), (10, 27, 1, 1, 32)]
    chunk, meta_bytes = L.hb_pack_chunk_elems(), L.hb_pack_meta_bytes()
    dt = np.dtype([("ptrs", "<u8", (3,)), ("ints", "<i4", (8,))])
    assert dt.itemsize == meta_bytes
    metas = np.zeros(len(shapes), dtype=dt)
    rows, keep, single = [], [], []
    for i, (cout, cin, r, s, cin_p) in enumerate(shapes):
        w = torch.randn(cout, r, s, cin, device="cuda")
        cout_p, cin_d = (cout + 15) // 16 * 16, (cin_p + 15) // 16 * 16
        need_d = i % 2 == 0
        wf = torch.full((cout_p, r, s, cin_p), float("nan"), device="cuda", dtype=torch.bfloat16)
        wd = torch.full((cin_d, r, s, cout_p), float("nan"), device="cuda", dtype=torch.bfloat16) if need_d else None
        wf1, wd1 = torch.empty_like(wf), (torch.empty_like(wd) if need_d else None)
        assert L.hb_pack_conv_weights(ptr(w), ptr(wf1), ptr(wd1), cout, cin, r, s, cin_p, cin_d, cout_p, cout_p, stream_ptr()) == 0
        metas[i]["ptrs"] = (w.data_ptr(), wf.data_ptr(), wd.data_ptr() if need_d else 0)
        metas[i]["ints"] = (cout, cin, r, s, cin_p, cin_d, cout_p, cout_p)
        nel = wf.numel() + (wd.numel() if need_d else 0)
        nch = (nel + chunk - 1) // chunk
        rows.append(np.stack([np.full(nch, i, dtype=np.int32), np.arange(nch, dtype=np.int32)], 1))
        keep.append((w, wf, wd))
        single.append((wf1, wd1))
    chunks = np.ascontiguousarray(np.concatenate(rows, 0))
    md = torch.from_numpy(metas.view(np.uint8).reshape(len(shapes), -1).copy()).cuda()
    cd = torch.from_numpy(chunks).cuda()
    assert L.hb_pack_conv_weights_multi(ptr(md), ptr(cd), int(chunks.shape[0]), stream_ptr()) == 0
    torch.cuda.synchronize()
    for (w, wf, wd), (wf1, wd1) in zip(keep, single):
        assert torch.equal(wf.view(torch.int16), wf1.view(torch.int16))
        if wd is not None:
            assert torch.equal(wd.view(torch.int16), wd1.view(torch.int16))


def test_filter_pack_table_follows_parameter_updates_and_moves():
    """The host-side packing cache (holocron_b200/nn/_fused.py::_PackTable): in-place parameter updates are picked up by
    ONE multi-tensor launch for all registered filters, and a parameter that moved to new storage is re-registered
    instead of being re-packed from its stale view. Scaling fp32 master weights by 2 is exact in bf16, so outputs must
    double exactly."""
    from holocron_b200.nn import _fused as K
    torch.manual_seed(0)
    convs = [torch.nn.Conv2d(16, 32, 3, padding=1, bias=False).cuda().to(memory_format=torch.channels_last) for _ in range(3)]
    x = torch.randn(2, 16, 8, 8, device="cuda")

    def run():
        with torch.no_grad():
            return [K.conv2d(x, c.weight, None, 1, 1).float() for c in convs]

    y0 = run()                                   # first use: every filter packed on its own and registered
    with torch.no_grad():
        for c in convs:
            c.weight.mul_(2.0)                   # in-place update: version bump, same storage
    before = lib().hb_launch_count()
    y1 = run()
    launches = lib().hb_launch_count() - before
    assert launches == 1 + len(convs)            # one multi-tensor packing launch + one convolution per layer
    for a, b in zip(y0, y1):
        assert torch.equal(b, 2 * a)
    with torch.no_grad():                        # move one parameter to fresh storage, then update all of them again
        convs[1].weight.data = (convs[1].weight.data * 0.5).clone(memory_format=torch.channels_last)
    y2 = run()
    assert torch.equal(y2[1], y0[1]) and torch.equal(y2[0], y1[0])
    with torch.no_grad():
        for c in convs:
            c.weight.mul_(2.0)
    y3 = run()
    for a, b in zip(y2, y3):
        assert torch.equal(b, 2 * a)
