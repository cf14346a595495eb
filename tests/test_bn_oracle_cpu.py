"""The fp64 restatement of tests/_bn_oracle.py against nn.BatchNorm2d + activation modules, its tie handling and kink
mask, and its geometry helper on hand-worked cases. Runs without a GPU."""
import copy

import pytest
import torch
from torch import nn

import _bn_oracle as O
from oracle.functional import hard_mish

MODULES = {0: nn.Identity, 1: nn.ReLU, 2: nn.ReLU6, 3: nn.SiLU, 4: lambda: nn.LeakyReLU(0.1), 5: nn.Mish}


def _act_module(code):
    if code == O.ACT_HARDMISH:
        return hard_mish
    return MODULES[code]()


def _rows(x):
    return x.permute(0, 2, 3, 1).reshape(-1, x.shape[1])


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("res", ["none", "inside", "after"])
@pytest.mark.parametrize("act", range(7))
@pytest.mark.parametrize("nb", [1, 2, 3])
def test_oracle_matches_batchnorm_modules(nb, act, res, train):
    torch.manual_seed(nb * 100 + act * 10 + len(res) + train)
    n, c, h, w = 2, 16, 5, 3
    bns = [nn.BatchNorm2d(c).double().train(train) for _ in range(nb)]
    for bn in bns:
        with torch.no_grad():
            bn.weight.uniform_(0.5, 2.0)
            bn.bias.normal_(0, 0.5)
            bn.running_mean.normal_(0, 1)
            bn.running_var.uniform_(0.5, 2.0)
    xs = [(torch.randn(n, c, h, w, dtype=torch.float64) * (b + 1) + b).requires_grad_(True) for b in range(nb)]
    r = torch.randn(n, c, h, w, dtype=torch.float64, requires_grad=True) if res != "none" else None
    d = torch.randn(n, c, h, w, dtype=torch.float64)
    # modules: what the fused path replaces
    running = None if train else [(bn.running_mean.clone(), bn.running_var.clone()) for bn in bns]
    mods = copy.deepcopy(bns)
    z = sum(bn(x) for bn, x in zip(mods, xs))
    if res == "inside":
        z = z + r
    out_m = _act_module(act)(z)
    if res == "after":
        out_m = out_m + r
    leaves = xs + ([r] if r is not None else []) + [p for bn in mods for p in (bn.weight, bn.bias)]
    g_m = torch.autograd.grad(out_m, leaves, d)
    # oracle on [M, C] rows
    xr = [_rows(x) for x in xs]
    out_o, _ = O.bn_act_ref(xr, [bn.weight for bn in bns], [bn.bias for bn in bns], act, 0.1,
                            _rows(r) if r is not None else None, res == "after", running)
    leaves_o = xs + ([r] if r is not None else []) + [p for bn in bns for p in (bn.weight, bn.bias)]
    g_o = torch.autograd.grad(out_o, leaves_o, _rows(d))
    torch.testing.assert_close(out_o, _rows(out_m), rtol=1e-12, atol=1e-12)
    for a, b in zip(g_o, g_m):
        torch.testing.assert_close(a, b, rtol=1e-10, atol=1e-12)


def test_oracle_act_only():
    x = torch.randn(64, 8, dtype=torch.float64)
    for code in range(7):
        out, z = O.bn_act_ref([], [], [], code, 0.1, x)
        assert torch.equal(z, x)
        ref = hard_mish(x) if code == O.ACT_HARDMISH else _act_module(code)(x)
        torch.testing.assert_close(out, ref, rtol=0, atol=1e-15)


def test_frelu_ties_split_evenly():
    u = torch.tensor([[1.0, 2.0, -3.0, 0.5]], dtype=torch.float64).repeat(4, 1)
    u[1:] += torch.randn(3, 4, dtype=torch.float64)
    r = u.clone()
    r[:, 1] = -5.0
    ur = u.clone().requires_grad_(True)
    rr = r.clone().requires_grad_(True)
    y = torch.maximum(ur, rr)
    gu, gr = torch.autograd.grad(y, (ur, rr), torch.ones_like(y))
    tie = u == r
    assert torch.equal(gu[tie], torch.full_like(gu[tie], 0.5)) and torch.equal(gr[tie], torch.full_like(gr[tie], 0.5))
    assert torch.equal(gu[:, 1], torch.ones(4, dtype=torch.float64)) and torch.equal(gr[:, 1], torch.zeros(4, dtype=torch.float64))
    # and through the oracle: an eval branch with scale exactly 1, shift exactly 0
    ones, zeros = torch.ones(4, dtype=torch.float64), torch.zeros(4, dtype=torch.float64)
    out, z = O.bn_act_ref([ur], [ones], [zeros], O.ACT_FRELU, 0.0, rr, running=[(zeros, ones - 2.0 ** -10)], eps=2.0 ** -10)
    assert torch.equal(out.detach(), torch.maximum(u, r))
    gu2, gr2 = torch.autograd.grad(out, (ur, rr), torch.ones_like(out))
    assert torch.equal(gu2, gu) and torch.equal(gr2, gr)


def test_kink_mask():
    z = torch.tensor([-2.05, -2.0, -1.99, -1.0, -1e-7, 0.0, 3e-7, 0.5, 5.9999999, 6.0, 6.2], dtype=torch.float64)
    dz = torch.full_like(z, 1e-6)
    near0 = [False, False, False, False, True, True, True, False, False, False, False]
    near6 = [False] * 8 + [True, True, False]
    near_m2 = [False, True] + [False] * 9
    for code, want in ((O.ACT_RELU, near0), (O.ACT_LEAKY, near0),
                       (O.ACT_RELU6, [a or b for a, b in zip(near0, near6)]),
                       (O.ACT_HARDMISH, [a or b for a, b in zip(near0, near_m2)]),
                       (O.ACT_NONE, [False] * 11), (O.ACT_SILU, [False] * 11), (O.ACT_MISH, [False] * 11)):
        assert O.kink_mask(code, z, dz).tolist() == want, code
    r = z + torch.tensor([0.0, 1e-7, -1e-5, 1.0, 0, 0, 0, 0, 0, 0, 2e-6], dtype=torch.float64)
    assert O.kink_mask(O.ACT_FRELU, z, dz, r).tolist() == [True, True, False, False] + [True] * 6 + [False]


@pytest.mark.parametrize("c,cg_t,rows_t,slabs", [(8, 1, 256, 1), (48, 6, 42, 1), (152, 19, 13, 1), (256, 32, 8, 1),
                                                 (264, 17, 15, 2), (304, 19, 13, 2), (1280, 32, 8, 5)])
def test_geometry(c, cg_t, rows_t, slabs):
    g = O.geometry(c)
    assert (g.cg_t, g.rows_t, g.slabs, g.cg_total) == (cg_t, rows_t, slabs, c // 8)
    # slabs cover the channel groups, the last one possibly ragged (264: 17 + 16)
    assert (g.slabs - 1) * g.cg_t < g.cg_total <= g.slabs * g.cg_t


def test_ring_depth_and_grid():
    assert [O.ring_depth(t) + 1 for t in (1, 2, 3, 4, 5)] == [8, 8, 4, 4, 4]
    # 1280 channels: 5 slabs, 132 SMs x 4 blocks -> 105 row blocks at most; 17672 rows of 8 lanes -> 2209 blocks wanted
    assert O.grid_rows(1280, 8 * 47 * 47, 132, 4) == 105
    assert O.rows_per_lane(1280, 8 * 47 * 47, 105) == 22
    assert O.grid_rows(48, 7, 132, 4) == 1 and O.rows_per_lane(48, 7, 1) == 1


def test_bounds_cover_a_float32_emulation_of_the_statistics():
    """Sequential fp32 lane sums of R rows, then fp64 over lanes: the mean / variance errors stay inside the bounds."""
    torch.manual_seed(0)
    m, lanes = 4099, 37
    for ratio in (0.0, 8.0, 64.0):
        u = (ratio + torch.randn(m, 3, dtype=torch.float64)).bfloat16().double()
        s = torch.zeros(lanes, 3, dtype=torch.float32)
        q = torch.zeros(lanes, 3, dtype=torch.float32)
        for i in range(m):
            f = u[i].float()
            s[i % lanes] += f
            q[i % lanes] += f * f
        mean = s.double().sum(0) / m
        var = q.double().sum(0) / m - mean * mean
        mu, v = O.batch_stats(u)
        dmean, dvar = O.stats_bounds(u, -(-m // lanes))
        assert bool(((mean - mu).abs() <= dmean).all()) and bool(((var - v).abs() <= dvar).all()), ratio
