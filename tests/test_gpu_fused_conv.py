"""GPU parity tests of the general tensor-core convolution launch (hb_conv2d_fused_bf16) and of the statistics /
gradient plumbing built on it:

  * dual output   - y3 = conv3x3(x), y1 = conv1x1(x) from ONE read of x (RepVGG forward, reference repvgg.py:71-73);
  * K extension   - dX = dgrad3x3(dY3) + dgrad1x1(dY1) + residual in one accumulator (RepVGG backward);
  * statistics    - per-channel (sum, sum of squares) partials from the convolution epilogue / the fused BatchNorm forward
                    pass == the sums of the stored bf16 tensor, summed in a fixed order: two runs are bit-identical;
  * direct gradients - weight and BatchNorm-parameter gradients ADDED into GradBucket views by the reduction kernels ==
                    what autograd accumulates without the bucket.

References are torch fp32 ops on the same bf16-rounded operands. Tolerances: bf16 outputs 4e-3 rel-L2 (output rounding),
fp32 statistics 1e-5, fp32 gradients 1e-3."""
import pytest
import torch
import torch.nn.functional as TF

from holocron_b200.distributed import GradBucket
from holocron_b200.models.classification.repvgg import RepBlock
from holocron_b200.nn import _fused as K

from _bounds import assert_within, conv_ref, epilogue_ref

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _cl(t):
    return t.cuda().to(torch.bfloat16).contiguous(memory_format=torch.channels_last)


def _stats_of(t):
    parts, slots = K.get_stats(t)
    return parts[:slots].double().sum(0)            # [C, 2]


def _ref_stats(t):
    tf = t.double()
    return torch.stack([tf.sum((0, 2, 3)), (tf * tf).sum((0, 2, 3))], 1)


DUAL_CASES = [
    # N, H, W, Cin, Cout, stride
    (2, 14, 14, 48, 48, 1),       # 3 of 4 k-steps in the only channel block
    (3, 28, 28, 96, 96, 1),       # 64 + 32 channels
    (2, 14, 14, 192, 192, 1),     # two Cout tiles of 96
    (2, 28, 28, 96, 192, 2),      # stride-2 stage entry
    (1, 14, 14, 192, 1280, 2),    # 10 Cout tiles, grid rounded to a multiple of 10
    (2, 7, 7, 1280, 1280, 1),
    (5, 9, 11, 16, 32, 1),        # ragged M tile
]


@pytest.mark.parametrize("case", DUAL_CASES)
def test_dual_output_conv_and_epilogue_statistics(case):
    n, h, w, cin, cout, stride = case
    torch.manual_seed(0)
    x = torch.randn(n, cin, h, w).bfloat16()
    w3 = (torch.randn(cout, cin, 3, 3) / (9 * cin) ** 0.5).bfloat16()
    w1 = (torch.randn(cout, cin, 1, 1) / cin ** 0.5).bfloat16()
    r3 = TF.conv2d(x.float(), w3.float(), None, stride, 1)
    r1 = TF.conv2d(x.float(), w1.float(), None, stride, 0)
    wf3 = w3.permute(0, 2, 3, 1).contiguous().cuda()
    wf1 = w1.permute(0, 2, 3, 1).contiguous().cuda()
    y3, y1 = K.conv2d_forward_raw(_cl(x), wf3, cout, 3, 3, stride, 1, 1, w2=wf1, want_stats=True)
    assert y3.shape == r3.shape and y1.shape == r1.shape
    assert rel_l2(y3, r3) < 4e-3 and rel_l2(y1, r1) < 4e-3
    assert_within(y3, *conv_ref(x, w3, None, stride, 1), "y3")
    assert_within(y1, *conv_ref(x, w1, None, stride, 0), "y1")
    # statistics are those of the STORED bf16 tensors
    assert rel_l2(_stats_of(y3), _ref_stats(y3)) < 1e-5
    assert rel_l2(_stats_of(y1), _ref_stats(y1)) < 1e-5
    # deterministic: a second launch gives bit-identical outputs and partials
    z3, z1 = K.conv2d_forward_raw(_cl(x), wf3, cout, 3, 3, stride, 1, 1, w2=wf1, want_stats=True)
    assert torch.equal(y3, z3) and torch.equal(y1, z1)
    p, s = K.get_stats(y3)
    q, t = K.get_stats(z3)
    assert s == t and torch.equal(p[:s], q[:t])


@pytest.mark.parametrize("case", [(2, 14, 14, 48, 48, 3), (2, 56, 56, 48, 48, 3), (2, 28, 28, 96, 96, 3), (2, 14, 14, 192, 192, 3),
                                  (2, 14, 14, 64, 128, 1), (3, 7, 7, 1280, 256, 1)])
def test_single_conv_statistics_all_paths(case):
    """Row-window kernel (C <= 64 .. 128 stride-1 3x3) and the generic kernel both emit correct statistics."""
    n, h, w, cin, cout, k = case
    torch.manual_seed(1)
    x = torch.randn(n, cin, h, w).bfloat16()
    wt = (torch.randn(cout, cin, k, k) / (k * k * cin) ** 0.5).bfloat16()
    ref = TF.conv2d(x.float(), wt.float(), None, 1, k // 2)
    y = K.conv2d_forward_raw(_cl(x), wt.permute(0, 2, 3, 1).contiguous().cuda(), cout, k, k, 1, k // 2, 1, want_stats=True)
    assert rel_l2(y, ref) < 4e-3
    assert_within(y, *conv_ref(x, wt, None, 1, k // 2), "y")
    assert rel_l2(_stats_of(y), _ref_stats(y)) < 1e-5


@pytest.mark.parametrize("case", [(2, 14, 14, 192, 192, True), (2, 28, 28, 96, 96, True), (2, 7, 7, 1280, 1280, False),
                                  (3, 14, 14, 48, 48, True), (2, 9, 11, 32, 16, False)])
def test_k_extension_with_residual(case):
    n, h, w, c, cd, with_res = case
    torch.manual_seed(2)
    d3, d1 = torch.randn(n, c, h, w).bfloat16(), torch.randn(n, c, h, w).bfloat16()
    w3 = (torch.randn(cd, c, 3, 3) / (9 * c) ** 0.5).bfloat16()
    w1 = (torch.randn(cd, c, 1, 1) / c ** 0.5).bfloat16()
    res = torch.randn(n, cd, h, w).bfloat16() if with_res else None
    ref = TF.conv2d(d3.float(), w3.float(), None, 1, 1) + TF.conv2d(d1.float(), w1.float())
    if with_res:
        ref = ref + res.float()
    y = K.conv2d_forward_raw(_cl(d3), w3.permute(0, 2, 3, 1).contiguous().cuda(), cd, 3, 3, 1, 1, 1, None,
                             _cl(res) if with_res else None, K.ACT_NONE, xe=_cl(d1), we=w1.permute(0, 2, 3, 1).contiguous().cuda())
    assert rel_l2(y, ref) < 4e-3
    r3, a3 = conv_ref(d3, w3, None, 1, 1)
    r1, a1 = conv_ref(d1, w1)
    ref, a, slack = epilogue_ref(r3 + r1, a3 + a1, res if with_res else None)
    assert_within(y, ref, a, "y", slack=slack)


def test_bn_forward_emits_output_statistics_and_is_deterministic():
    torch.manual_seed(3)
    n, c, h, w = 4, 96, 28, 28
    u = [_cl(torch.randn(n, c, h, w)) for _ in range(3)]
    bns = [torch.nn.BatchNorm2d(c).cuda().train() for _ in range(3)]
    for bn in bns:
        torch.nn.init.uniform_(bn.weight, 0.5, 1.5)
        torch.nn.init.uniform_(bn.bias, -0.5, 0.5)
    out = K.bn_act(u, bns, K.ACT_RELU, 0.0, emit_stats=True)
    ref = sum(TF.batch_norm(t.float(), None, None, bn.weight, bn.bias, True, 0.1, bn.eps) for t, bn in zip(u, bns)).relu()
    assert rel_l2(out, ref) < 4e-3
    assert rel_l2(_stats_of(out), _ref_stats(out)) < 1e-5
    # running statistics followed nn.BatchNorm2d (momentum 0.1, unbiased variance)
    m = n * h * w
    for t, bn in zip(u, bns):
        tf = t.float()
        assert rel_l2(bn.running_mean, 0.1 * tf.mean((0, 2, 3))) < 1e-3
        assert rel_l2(bn.running_var, 0.9 + 0.1 * tf.var((0, 2, 3), unbiased=True)) < 1e-4
        assert int(bn.num_batches_tracked) == 1
    out2 = K.bn_act(u, bns, K.ACT_RELU, 0.0, emit_stats=True)
    assert torch.equal(out, out2)
    # backward: two runs bit-identical (fixed-order reductions, no atomics)
    grads = []
    for _ in range(2):
        us = [t.clone().requires_grad_(True) for t in u]
        for bn in bns:
            bn.weight.grad = bn.bias.grad = None
        o = K.bn_act(us, bns, K.ACT_RELU, 0.0)
        o.backward(torch.ones_like(o) * 0.5)
        grads.append([t.grad.clone() for t in us] + [bn.weight.grad.clone() for bn in bns] + [bn.bias.grad.clone() for bn in bns])
    assert all(torch.equal(a, b) for a, b in zip(*grads))


@pytest.mark.parametrize("cfg", [(48, 48, 1, True, 28), (96, 96, 1, True, 14), (192, 192, 1, True, 14), (48, 96, 2, False, 28),
                                 (192, 1280, 2, False, 14)])
def test_repblock_direct_gradients_match_autograd_accumulation(cfg):
    """Same block, same input: gradients added by the kernels into GradBucket views == gradients accumulated by autograd."""
    cin, cout, stride, ident, hw = cfg
    torch.manual_seed(4)
    x = torch.randn(4, cin, hw, hw)
    up = torch.randn(4, cout, hw // stride, hw // stride)
    blocks = []
    for direct in (False, True):
        torch.manual_seed(5)
        blk = RepBlock(cin, cout, stride, ident).cuda().to(memory_format=torch.channels_last).train()
        for p in blk.parameters():
            if p.ndim == 1:
                torch.nn.init.uniform_(p, 0.5, 1.5)
        bucket = GradBucket(blk.parameters(), direct=direct)
        xin = x.cuda().requires_grad_(True)
        for _ in range(2):          # two backward passes: gradients ACCUMULATE in both modes
            y = blk(xin)
            (y.float() * up.cuda()).sum().backward()
        blocks.append((blk, bucket, xin.grad.clone(), y.detach().clone()))
    (b0, _, gx0, y0), (b1, _, gx1, y1) = blocks
    assert torch.equal(y0, y1)
    assert rel_l2(gx1, gx0) < 1e-6
    for (n0, p0), (n1, p1) in zip(b0.named_parameters(), b1.named_parameters()):
        assert p1.grad is not None and rel_l2(p1.grad, p0.grad) < 1e-5, n0


REPBLOCK_DX_CASES = [
    # Cin, Cout, stride, H, W
    (32, 64, 2, 1, 7),       # stride 2 on a one-pixel side: zero insertion + convolution instead of parity classes
    (32, 64, 2, 6, 1),
    (24, 48, 2, 1, 5),       # the same with the input channels padded to 32
    (3, 32, 1, 12, 12),      # padded input channels and an input that needs its gradient: no im2col stem
    (3, 32, 2, 12, 12),
    (24, 48, 1, 10, 10),
    (24, 48, 2, 10, 10),
]


@pytest.mark.parametrize("case", REPBLOCK_DX_CASES)
def test_repblock_input_gradient_paths_vs_fp32(case):
    """Input-gradient paths of the fused RepBlock that the RepVGG widths never take: output, input gradient and parameter
    gradients against the same block in fp32 torch ops, on bf16-representable inputs and filters. The reference's ReLU
    takes the fused block's mask, so that a pre-activation rounding to the other side of zero in bf16 (a full upstream
    gradient switched on or off) is not counted as an error. Tolerances as in test_gpu_repvgg.py's golden block."""
    from oracle.models import RepBlockOracle
    cin, cout, stride, h, w = case
    torch.manual_seed(7)
    blk = RepBlock(cin, cout, stride, False).train()
    with torch.no_grad():
        for p in blk.parameters():
            if p.ndim == 1:
                torch.nn.init.uniform_(p, 0.5, 1.5)
            else:
                p.copy_(p.bfloat16().float())
    ref = RepBlockOracle(cin, cout, stride, False).train()
    ref.load_state_dict(blk.state_dict())
    x = torch.randn(4, cin, h, w).bfloat16().float()
    blk = blk.cuda()
    xd = x.cuda().requires_grad_(True)
    y = blk(xd)
    up = torch.randn(y.shape)
    (y.float() * up.cuda()).sum().backward()
    xo = x.clone().requires_grad_(True)
    z = sum(b(xo) for b in ref.branches)
    yo = z.relu()
    (z * (y.float().cpu() > 0) * up).sum().backward()
    assert y.shape == yo.shape
    assert rel_l2(y, yo) < 6e-3
    assert rel_l2(xd.grad, xo.grad) < 2e-2
    ref_params = dict(ref.named_parameters())
    for name, p in blk.named_parameters():
        assert p.grad is not None and rel_l2(p.grad, ref_params[name].grad) < 2e-2, name


def test_repblock_two_forward_backward_runs_are_bit_identical():
    torch.manual_seed(6)
    blk = RepBlock(96, 96, 1, True).cuda().to(memory_format=torch.channels_last).train()
    x = torch.randn(8, 96, 28, 28).cuda()
    runs = []
    for _ in range(2):
        for p in blk.parameters():
            p.grad = None
        xin = x.clone().requires_grad_(True)
        y = blk(xin)
        y.float().square().mean().backward()
        runs.append([y.detach().clone(), xin.grad.clone()] + [p.grad.clone() for p in blk.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*runs))
