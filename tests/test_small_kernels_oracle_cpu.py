"""The oracles of tests/_small_kernels_oracle.py on the CPU: they reproduce the goldens the unmodified reference wrote, the
fp64 restatement of the box backward equals torch autograd of the reference's box operators on tie-heavy integer boxes,
and the case tables of tests/test_gpu_small_kernels_bounds.py reach every launch path of the four kernel families."""
import pytest
import torch

import _small_kernels_oracle as O
from conftest import load_golden

SMS_RANGE = (100, 114, 132, 144)   # H100 PCIe has 114 SMs, SXM 132


def test_activation_oracles_match_golden():
    g = load_golden("activations")
    x = g["x"].double()
    ones = torch.ones_like(x)
    assert torch.allclose(O.hard_mish_ref(x), g["hard_mish"].double(), rtol=1e-6, atol=1e-7)
    assert torch.allclose(O.hard_mish_grad_ref(x, ones), g["hard_mish_grad"].double(), rtol=1e-6, atol=1e-7)
    for beta in (1.0, 0.5):
        assert torch.allclose(O.nl_relu_ref(x, beta), g[f"nl_relu_b{beta}"].double(), rtol=1e-6, atol=1e-7)
        assert torch.allclose(O.nl_relu_grad_ref(x, ones, beta), g[f"nl_relu_b{beta}_grad"].double(), rtol=1e-6,
                              atol=1e-7)
        y = O.nl_relu_ref(x, beta)
        assert torch.allclose(O.nl_relu_grad_from_out_ref(y, ones, beta), O.nl_relu_grad_ref(x, ones, beta))


def test_activation_oracles_match_autograd_on_special_values():
    """NaN, +-inf and the clamp ends, against autograd of the reference compositions in fp64."""
    x = torch.tensor([float("nan"), float("inf"), -float("inf"), -2.0, 0.0, -1.0, 3.0, -3.0, 1e-30], dtype=torch.float64)
    dy = torch.linspace(0.5, 1.5, x.numel(), dtype=torch.float64)
    a = x.clone().requires_grad_(True)
    (0.5 * a * (a + 2).clamp(min=0, max=2)).backward(dy)
    torch.testing.assert_close(O.hard_mish_grad_ref(x, dy), a.grad, equal_nan=True)
    for beta in (1.0, 0.5):
        a = x.clone().requires_grad_(True)
        torch.log(1 + beta * torch.relu(a)).backward(dy)
        torch.testing.assert_close(O.nl_relu_grad_ref(x, dy, beta), a.grad, equal_nan=True)
        torch.testing.assert_close(O.nl_relu_ref(x, beta), torch.log(1 + beta * torch.relu(x)), equal_nan=True)
    torch.testing.assert_close(O.hard_mish_ref(x), 0.5 * x * (x + 2).clamp(min=0, max=2), equal_nan=True)


def test_dropblock_oracle_matches_golden():
    g = load_golden("convs")
    mask, kept = O.dropblock_mask_ref(g["dropblock_noise"], 0.3 / 9, 3)
    out = O.dropblock_out_ref(g["dropblock_x"], mask, kept)
    assert torch.allclose(out, g["dropblock_out"].double(), rtol=1e-6, atol=1e-7)
    # the reference's own op sequence in fp32 reproduces the golden bit for bit
    ref = O.dropblock_reference_ops(g["dropblock_x"], g["dropblock_noise"], 0.3 / 9, 3)
    assert torch.equal(ref, g["dropblock_out"])


def test_dropblock_scale_rounds_twice_in_the_reference():
    """numel / kept as the reference computes it is fl(fl(1 / kept) * numel), which differs from the once-rounded
    quotient for some counts: the rounding the fp32 kernels restate."""
    numel = 2 * 56 * 56
    k = torch.arange(1, numel + 1, dtype=torch.float32)
    ref = numel / k[:, None].sum(1)          # the reference's `int / Tensor`
    twice = (torch.ones_like(k) / k) * numel
    once = (torch.full_like(k, numel, dtype=torch.float64) / k.double()).float()
    assert torch.equal(ref, twice)
    assert int((twice != once).sum()) > 0


@pytest.mark.parametrize("mode", [O.IOU, O.GIOU, O.PENALTY, O.DIOU])
def test_pair_grad_matches_autograd_on_integer_boxes(mode):
    gen = torch.Generator().manual_seed(100 + mode)
    for trial in range(60):
        border = 5 if trial % 3 == 0 else 0
        b1 = O.integer_boxes(6, gen, border=border)
        b2 = torch.cat([O.integer_boxes(4, gen, border=border), b1[:2]])   # identical pairs too
        gout = torch.randn(6, 6, generator=gen, dtype=torch.float64)
        g1, g2, bound1, bound2 = O.box_grads_ref(mode, b1, b2, gout)
        a1, a2 = O.box_autograd(mode, b1, b2, gout)
        torch.testing.assert_close(g1, a1, rtol=1e-12, atol=1e-12, equal_nan=True)
        torch.testing.assert_close(g2, a2, rtol=1e-12, atol=1e-12, equal_nan=True)
        fin = torch.isfinite(g1)
        assert bool((bound1[fin] >= 0).all())


def test_pair_grad_matches_box_goldens():
    g = load_golden("boxes")
    b1, b2, up = g["b1"], g["b2"], g["up"]
    ones = torch.ones(b1.shape[0], b2.shape[0], dtype=torch.float64)
    for mode, key in ((O.GIOU, "box_giou"), (O.DIOU, "diou_loss"), (O.DIOU, "ciou_loss")):
        g1, g2, bound1, bound2 = O.box_grads_ref(mode, b1, b2, ones)
        assert bool(((g1 - g[f"rnd_{key}_grad1"].double()).abs() <= 4 * bound1 + 1e-7).all())
        assert bool(((g2 - g[f"rnd_{key}_grad2"].double()).abs() <= 4 * bound2 + 1e-7).all())
    g1, g2, _, _ = O.box_grads_ref(O.DIOU, b1, b2, up)
    torch.testing.assert_close(g1, g["rnd_ciou_wgrad1"].double(), rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(g2, g["rnd_ciou_wgrad2"].double(), rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("sms", SMS_RANGE)
def test_activation_case_routes(sms):
    reached = set()
    for name, nvec, tail, aligned, route in O.ACT_CASES:
        for dtype in (torch.float32, torch.bfloat16, torch.float16):
            n = nvec * O.vec_width(dtype) + tail
            for binary in (False, True):
                got = O.route_act(n, dtype, binary, aligned, sms)
                assert got == frozenset(route), (name, dtype, binary, sorted(got))
                reached |= got
    assert reached == set(O.ACT_PATHS)


@pytest.mark.parametrize("sms", SMS_RANGE)
def test_dropblock_case_routes(sms):
    reached = set()
    for dtype in (torch.float32, torch.bfloat16, torch.float16):
        for name, n, c, h, w, cl, offset, inplace, route in O.DB_APPLY_CASES:
            got = O.route_dropblock(n, c, h, w, dtype, cl, offset == 0, sms)
            assert got == frozenset(route), (name, dtype, sorted(got))
            reached |= got
    n, c, h, w, route = O.DB_BIG
    assert n * h * w > 2 ** 24
    got = O.route_dropblock(n, c, h, w, torch.float32, False, True, sms)
    assert got == frozenset(route)
    reached |= got
    assert reached == set(O.DB_PATHS)


@pytest.mark.parametrize("sms", SMS_RANGE)
def test_gap_case_routes(sms):
    reached = set()
    for n, hw, c, route in O.GAP_CASES:
        got = O.route_gap(n, hw, c, sms)
        assert got == frozenset(route), (n, hw, c, sorted(got))
        reached |= got
    assert reached == set(O.GAP_PATHS)
    cs = {c for _, _, c, _ in O.GAP_CASES}
    assert {8, 24, 1280, 2048} <= cs
    assert {1, 3136} <= {hw for _, hw, _, _ in O.GAP_CASES}
    assert any(hw % 2 == 1 and hw > 1 for _, hw, _, _ in O.GAP_CASES)


def test_gap_chain_counts_rows_and_fold():
    # C = 8: one channel group, 256 row lanes; 600 rows -> lane 0 owns rows 0, 256, 512: one pair and a lone row
    assert O.slab_geo(8) == (1, 1, 256, 1)
    assert O.gap_chain(600, 8) == 2 * 1 + 1 + 255 + 2
    assert O.slab_geo(264) == (33, 17, 15, 2)


def test_box_case_routes():
    reached = set()
    for name, m, n, want, route in O.BOX_SIZES:
        got = O.route_box(m, n, *want)
        assert got == frozenset(route), (name, sorted(got))
        reached |= got
    assert reached == set(O.BOX_PATHS)
