"""CPU emulation of the bf16 storage of the fused LambdaLayer path, against the reference's fixture
(tests/golden/lambda_layer.pt). The fp32 restatement is rounded to bf16 wherever the GPU path stores a tensor (input,
projection weights and outputs, BatchNorm outputs, layer output, and every gradient at those points). The rel-L2 it
reaches is what bf16 storage alone costs; it sizes the one bound of tests/test_gpu_lambda.py that is looser than 1e-2."""
import pytest
import torch
import torch.nn.functional as F

import holocron_b200 as hb

import _lambda_oracle as O
from conftest import load_golden


class _RoundBF16(torch.autograd.Function):
    """bf16 rounding of a value and of its gradient."""

    @staticmethod
    def forward(ctx, x):
        return x.bfloat16().float()

    @staticmethod
    def backward(ctx, g):
        return g.bfloat16().float()


def _emulated_grads(case):
    rb = _RoundBF16.apply
    c, o, dk, n, r, heads, u = case["cfg"]
    torch.manual_seed(case["seed"])
    mod = hb.nn.LambdaLayer(c, o, dk, n=n, r=r, num_heads=heads, dim_u=u)
    x = case["x"].clone().requires_grad_(True)

    def bn(t, m):
        return F.batch_norm(t, None, None, m.weight, m.bias, True, 0.0, m.eps)

    xb = rb(x)
    q = rb(bn(rb(F.conv2d(xb, rb(mod.to_q.weight))), mod.norm_q))
    k = rb(F.conv2d(xb, rb(mod.to_k.weight)))
    v = rb(bn(rb(F.conv2d(xb, rb(mod.to_v.weight))), mod.norm_v))
    y = rb(O.lambda_core(q, k, v, mod.R if r else mod.pos_emb, dk, u, heads, r))
    torch.manual_seed(case["w_seed"])
    (y * torch.randn(case["y"].shape)).sum().backward()
    return {name: p.grad for name, p in mod.named_parameters()}


def _rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


@pytest.fixture(scope="module")
def g():
    return load_golden("lambda_layer")


def test_bf16_storage_alone_exceeds_1e2_on_norm_v_weight(g):
    """On the in_channels = 3 configuration, bf16 storage alone puts norm_v.weight's gradient above 1e-2 (1.09e-2) and
    below the 2e-2 bar the GPU fixture test holds it to; every other parameter stays within 1e-2 on every case."""
    worst = {}
    for case in g["cases"]:
        for name, grad in _emulated_grads(case).items():
            err = _rel_l2(grad, case["grads"][name])
            worst[name] = max(worst.get(name, 0.0), err)
    assert 1e-2 < worst["norm_v.weight"] <= 2e-2, worst["norm_v.weight"]
    assert all(err <= 1e-2 for name, err in worst.items() if name != "norm_v.weight"), worst
