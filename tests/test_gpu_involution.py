"""Involution2d on the H100: the three involution kernels against an fp64 restatement fed the same bf16 values, the module
against the reference's fixture (tests/golden/involution.pt), the reference's own test shapes, determinism and CUDA-graph
replay."""
import pytest
import torch

import holocron_b200 as hb
from holocron_b200._lib import lib, ptr, stream_ptr
from holocron_b200.nn import _fused as K
from holocron_b200.nn._involution import involution2d

import _involution_oracle as O
from _bounds import assert_within as _assert_within
from conftest import load_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _cl(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous(memory_format=torch.channels_last)


def _check_kernels(n, c, g, k, s, d, p, h, w, seed=0):
    torch.manual_seed(seed)
    ho = (h + 2 * p - d * (k - 1) - 1) // s + 1
    wo = (w + 2 * p - d * (k - 1) - 1) // s + 1
    kp = K.round_up(g * k * k, 16)
    x = _cl(torch.randn(n, c, h, w, device=DEV).bfloat16()).requires_grad_(True)
    ker = _cl(torch.randn(n, kp, ho, wo, device=DEV).bfloat16()).requires_grad_(True)
    dy = _cl(torch.randn(n, c, ho, wo, device=DEV).bfloat16())
    y = involution2d(x, ker, k, s, p, d, g)
    y.backward(dy)
    # fp64 on the same bf16 values; the same computation on absolute values bounds the cancellation
    x64, k64 = x.detach().double().requires_grad_(True), ker.detach().double().requires_grad_(True)
    ref = O.involution2d(x64, k64, k, s, p, d, g)
    ref.backward(dy.double())
    xa, ka = x.detach().double().abs().requires_grad_(True), ker.detach().double().abs().requires_grad_(True)
    refa = O.involution2d(xa, ka, k, s, p, d, g)
    refa.backward(dy.double().abs())
    _assert_within(y.detach(), ref.detach(), refa.detach(), "y")
    _assert_within(x.grad, x64.grad, xa.grad, "dx")
    _assert_within(ker.grad, k64.grad, ka.grad, "dker")
    assert torch.equal(ker.grad[:, g * k * k:], torch.zeros_like(ker.grad[:, g * k * k:])), "dker padding columns"
    assert y.dtype == torch.bfloat16 and (c % 8 or y.is_contiguous(memory_format=torch.channels_last))


# (C, G): uniform vectors with 1, 2 and 3 vectors per group, mixed vectors with and without channel padding
GROUPS = [(8, 1), (12, 6), (16, 4), (48, 2), (64, 4), (256, 16)]


@pytest.mark.parametrize("cg", GROUPS, ids=[f"C{c}G{g}" for c, g in GROUPS])
@pytest.mark.parametrize("k", [1, 3, 5, 7])
@pytest.mark.parametrize("s", [1, 2, 3])
@pytest.mark.parametrize("d", [1, 2])
def test_kernels_vs_fp64(cg, k, s, d):
    c, g = cg
    _check_kernels(2, c, g, k, s, d, (k // 2) * d, 11, 9, seed=k * 100 + s * 10 + d)


def test_kernels_unpadded_and_wide_halo():
    # padding 0; and a dilation whose halo box does not fit the shared-memory tile (global-memory taps)
    _check_kernels(2, 64, 4, 3, 1, 1, 0, 13, 10)
    _check_kernels(1, 16, 2, 7, 3, 6, 5, 40, 37)
    _check_kernels(1, 12, 6, 7, 3, 6, 5, 40, 37)


def test_kernels_rednet_layer():
    _check_kernels(8, 256, 16, 7, 1, 1, 3, 28, 28)


@pytest.mark.parametrize("c,g", [(12, 6), (20, 5)])
def test_padded_channels_are_zero(c, g):
    """The raw entry points write zeros into channels C..Cp-1 of y and dx, whatever the padded inputs hold."""
    torch.manual_seed(1)
    n, h, w, k = 2, 9, 7, 3
    cp, kp = K.round_up(c, 8), K.round_up(g * 9, 16)
    x = _cl(torch.randn(n, cp, h, w, device=DEV).bfloat16())
    ker = _cl(torch.randn(n, kp, h, w, device=DEV).bfloat16())
    dy = _cl(torch.randn(n, cp, h, w, device=DEV).bfloat16())
    y = torch.full_like(x, float("nan"))
    dx = torch.full_like(x, float("nan"))
    args = (n, h, w, c, cp, kp, k, g, 1, 1, 1, stream_ptr())
    assert lib().hb_involution_fwd_bf16(ptr(x), ptr(ker), ptr(y), *args) == 0
    assert lib().hb_involution_bwd_data_bf16(ptr(dy), ptr(ker), ptr(dx), *args) == 0
    torch.cuda.synchronize()
    assert torch.equal(y[:, c:], torch.zeros_like(y[:, c:]))
    assert torch.equal(dx[:, c:], torch.zeros_like(dx[:, c:]))
    assert torch.isfinite(y[:, :c]).all() and torch.isfinite(dx[:, :c]).all()


def _rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def _module_from_case(case):
    c, k, p, s, d, g, r = case["cfg"]
    mod = hb.nn.Involution2d(c, k, padding=p, stride=s, groups=g, dilation=d, reduction_ratio=r)
    mod.load_state_dict(case["init"])
    return mod.to(DEV)


def test_module_vs_fixture():
    gold = load_golden("involution")
    for case in gold["cases"]:
        mod = _module_from_case(case)
        x = case["x"].to(DEV).requires_grad_(True)
        y = mod(x)
        assert y.dtype == torch.float32 and y.shape == case["y"].shape
        (y * case["w"].to(DEV)).sum().backward()
        assert _rel_l2(y.detach().cpu(), case["y"]) <= 1e-2, case["cfg"]
        assert _rel_l2(x.grad.cpu(), case["dx"]) <= 1e-2, case["cfg"]
        for name, prm in mod.named_parameters():
            # reduce.bias sums the bf16 gradient of the reduce output over every pixel, and the terms cancel: a CPU
            # run of the fp32 formulation rounded to bf16 where this path stores tensors lands at 1.5e-2 on C = 24
            bar = 2e-2 if name == "reduce.bias" else 1e-2
            assert _rel_l2(prm.grad.cpu(), case["grads"][name]) <= bar, (case["cfg"], name)


@pytest.mark.parametrize("stride,out", [(1, 16), (2, 8)])
def test_reference_test_shapes(stride, out):
    """The shapes of the reference's own test_involution2d: (2, 8, 16, 16) in, K = 3, padding 1, reduction 2."""
    torch.manual_seed(0)
    mod = hb.nn.Involution2d(8, 3, 1, stride, reduction_ratio=2).to(DEV)
    x = torch.rand(2, 8, 16, 16, device=DEV, requires_grad=True)
    y = mod(x)
    assert y.shape == (2, 8, out, out)
    y.sum().backward()
    ref = O.involution_module(x.detach(), mod)
    assert _rel_l2(y.detach(), ref.detach()) <= 1e-2
    assert x.grad is not None and torch.isfinite(x.grad).all()


def test_bf16_channels_last_in_and_out():
    torch.manual_seed(0)
    mod = hb.nn.Involution2d(64, 7, 3, 1, 4, reduction_ratio=4).to(DEV)
    x = _cl(torch.randn(2, 64, 14, 14, device=DEV).bfloat16())
    y = mod(x)
    assert y.dtype == torch.bfloat16 and y.is_contiguous(memory_format=torch.channels_last)


def _run(mod, x, w):
    mod.zero_grad(set_to_none=True)
    x.grad = None
    y = mod(x)
    (y * w).sum().backward()
    return [y.detach().clone(), x.grad.clone()] + [p.grad.clone() for p in mod.parameters()]


@pytest.mark.parametrize("cfg", [(64, 7, 3, 1, 1, 4, 4), (64, 7, 3, 2, 1, 4, 4), (12, 3, 1, 1, 1, 6, 1.5)])
def test_deterministic_and_graph_replay(cfg):
    c, k, p, s, d, g, r = cfg
    torch.manual_seed(0)
    mod = hb.nn.Involution2d(c, k, padding=p, stride=s, groups=g, dilation=d, reduction_ratio=r).to(DEV)
    x = _cl(torch.randn(4, c, 16, 16, device=DEV).bfloat16()).requires_grad_(True)
    w = torch.randn(4, c, 16 // s, 16 // s, device=DEV).bfloat16()
    first, second = _run(mod, x, w), _run(mod, x, w)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _run(mod, x, w)
    torch.cuda.current_stream().wait_stream(side)
    mod.zero_grad(set_to_none=True)
    x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = mod(x)
        (y * w).sum().backward()
    graph.replay()
    torch.cuda.synchronize()
    replayed = [y, x.grad] + [p_.grad for p_ in mod.parameters()]
    for a, b in zip(first, replayed):
        assert torch.equal(a, b)
