"""LambdaLayer on the H100: the lambda kernels against an fp64 restatement fed the same bf16 values, the module against the
reference's fixture (tests/golden/lambda_layer.pt), the reference's own test shapes, determinism, CUDA-graph replay and
peak memory against the eager formulation."""
import pytest
import torch

import holocron_b200 as hb
from holocron_b200.nn import _fused as K
from holocron_b200.nn._lambda import lambda_layer

import _lambda_oracle as O
from _bounds import assert_within as _assert_within
from conftest import load_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _padded(b, c, h, w, scale=1.0):
    """bf16 channels_last [b, round_up(c, 8), h, w] with zero padding channels."""
    t = torch.zeros(b, K.round_up(c, 8), h, w, device=DEV)
    t[:, :c] = torch.randn(b, c, h, w, device=DEV) * scale
    return t.bfloat16().contiguous(memory_format=torch.channels_last)


def _dk_abs_terms(qa, k64, va, dya, dk, u, heads):
    """sigma_m * (a_m + sum_m' sigma a_m') per key channel, a_m = sum_v |dlc|[k,v] |v|[m,v*u+u'], |dlc| = sum |q| |dy|."""
    b, _, h, w = qa.shape
    n = h * w
    dv = va.shape[1] // u
    sig = k64.reshape(b, dk, u, n).softmax(-1)
    dlca = torch.einsum("bhkn,bhvn->bkv", qa.reshape(b, heads, dk, n), dya[:, :heads * dv].reshape(b, heads, dv, n))
    a = torch.einsum("bkv,bvum->bkum", dlca, va.reshape(b, dv, u, n))
    return (sig * (a + (sig * a).sum(-1, keepdim=True))).reshape(b, dk * u, h, w)


def _check_kernels(b, h, w, dk, u, heads, dv, r, seed=0):
    torch.manual_seed(seed)
    cq, ck, cv = heads * dk, dk * u, dv * u
    q, k, v = _padded(b, cq, h, w), _padded(b, ck, h, w, 2.0), _padded(b, cv, h, w)
    pos = (torch.randn(dk, u, 1, r, r, device=DEV) if r else torch.randn(h * w, h * w, dk, u, device=DEV) * 0.2)
    pos = pos.bfloat16().float().requires_grad_(True)
    for t in (q, k, v):
        t.requires_grad_(True)
    y = lambda_layer(q, k, v, pos, dk, u, heads, dv, r)
    dy = torch.randn(y.shape, device=DEV).bfloat16()
    y.backward(dy)
    rr = r or None
    # fp64 on the same bf16 values; the same computation on absolute values bounds the cancellation
    q64, k64, v64, p64 = (t.detach()[:, :c].double().requires_grad_(True) for t, c in ((q, cq), (k, ck), (v, cv), (pos, None)))
    ref = O.lambda_core(q64, k64, v64, p64, dk, u, heads, rr)
    ref.backward(dy.double())
    qa, va, pa = (t.detach()[:, :c].double().abs().requires_grad_(True) for t, c in ((q, cq), (v, cv), (pos, None)))
    ka = k.detach()[:, :ck].double().requires_grad_(True)
    refa = O.lambda_core(qa, ka, va, pa, dk, u, heads, rr)
    refa.backward(dy.double().abs())
    _assert_within(y.detach(), ref.detach(), refa.detach(), "y")
    _assert_within(q.grad[:, :cq], q64.grad, qa.grad, "dq")
    # dv and dR take the per-position gradient of the position lambda through a bf16 transient: 2^-8 of the terms
    _assert_within(v.grad[:, :cv], v64.grad, va.grad, "dv", rel=4e-3)
    _assert_within(pos.grad, p64.grad, pa.grad, "dpos", rel=4e-3)
    # dk = sigma_m * (dsigma_m - sum_m' sigma dsigma) with dsigma_m = sum_v dlc[k,v] * v[m,v*u+u'] in fp32 (no bf16
    # transient): each element within one ulp + 1e-5 * sigma_m * (|dsigma|_m + sum_m' sigma |dsigma|), the absolute terms
    # taken in fp64 with dlc over |q| |dy|
    _assert_within(k.grad[:, :ck], k64.grad, _dk_abs_terms(qa.detach(), k64.detach(), va.detach(), dy.double().abs(),
                                                          dk, u, heads), "dk")
    for t, c in ((q, cq), (k, ck), (v, cv)):
        assert torch.equal(t.grad[:, c:], torch.zeros_like(t.grad[:, c:])), "padding channels of the gradients"
    assert y.dtype == torch.bfloat16 and y.shape == (b, heads * dv, h, w)


# (dk, u, heads, dv, r): every dim_k, dim_u 1-4, 1-8 heads, dim_v with and without % 8, r from 1 to 23 and the global variant
GRID = [
    (8, 1, 1, 8, 1), (16, 1, 4, 8, 3), (32, 1, 2, 16, 5), (16, 2, 4, 12, 7), (8, 3, 3, 5, 3), (16, 4, 8, 8, 9),
    (32, 4, 1, 3, 11), (8, 1, 4, 64, 13), (16, 1, 4, 32, 23), (8, 2, 2, 24, 21), (16, 1, 6, 7, 15),
    (8, 1, 4, 8, 0), (16, 2, 2, 12, 0), (32, 4, 3, 5, 0),
]


@pytest.mark.parametrize("cfg", GRID, ids=[f"dk{a}u{b}h{c}v{d}r{e}" for a, b, c, d, e in GRID])
def test_kernels_vs_fp64(cfg):
    dk, u, heads, dv, r = cfg
    h, w = (5, 6) if r == 0 else (11, 9)
    _check_kernels(2, h, w, dk, u, heads, dv, r, seed=sum(cfg))


def test_kernels_lambdaresnet_layer():
    _check_kernels(2, 28, 28, 16, 1, 4, 32, 23)


def _rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def _module_from_case(case):
    c, o, dk, n, r, heads, u = case["cfg"]
    mod = hb.nn.LambdaLayer(c, o, dk, n=n, r=r, num_heads=heads, dim_u=u)
    mod.load_state_dict(case["init"])
    return mod.to(DEV)


def test_module_vs_fixture():
    gold = load_golden("lambda_layer")
    for case in gold["cases"]:
        mod = _module_from_case(case)
        x = case["x"].to(DEV).requires_grad_(True)
        y = mod(x)
        assert y.dtype == torch.float32 and y.shape == case["y"].shape
        torch.manual_seed(case["w_seed"])
        w = torch.randn(case["y"].shape)
        (y * w.to(DEV)).sum().backward()
        cfg = case["cfg"]
        assert _rel_l2(y.detach().cpu(), case["y"]) <= 1e-2, cfg
        assert _rel_l2(x.grad.cpu(), case["dx"]) <= 1e-2, cfg
        for name, prm in mod.named_parameters():
            # norm_v.weight sums the bf16 gradient of v times the normalised v over every position: a CPU run of the fp32
            # formulation rounded to bf16 where this path stores tensors lands at 1.09e-2 on in_channels = 3
            bar = 2e-2 if name == "norm_v.weight" else 1e-2
            assert _rel_l2(prm.grad.cpu(), case["grads"][name]) <= bar, (cfg, name)
        sd = mod.state_dict()
        for name, ref in case["running"].items():
            if name.endswith("num_batches_tracked"):
                assert int(sd[name]) == int(ref), (cfg, name)
            else:
                assert _rel_l2(sd[name].cpu(), ref) <= 1e-2, (cfg, name)
        mod.eval()
        with torch.no_grad():
            ye = mod(case["x"][:1].to(DEV))
        assert _rel_l2(ye.cpu(), case["y_eval"]) <= 1e-2, cfg


def test_refused_input_grid():
    gold = load_golden("lambda_layer")
    for err in gold["errors"]:
        assert err["raised"] == "RuntimeError"
        c, o, dk, n, r, heads, u = err["cfg"]
        mod = hb.nn.LambdaLayer(c, o, dk, n=n, r=r, num_heads=heads, dim_u=u).to(DEV)
        with pytest.raises(RuntimeError):
            mod(torch.randn(*err["shape"], device=DEV))


def test_reference_test_shapes():
    """The reference's own test_lambdalayer: LambdaLayer(8, 32, 16, r=13) on (2, 8, 32, 32), backward included."""
    torch.manual_seed(0)
    mod = hb.nn.LambdaLayer(8, 32, 16, r=13).to(DEV)
    x = torch.rand(2, 8, 32, 32, device=DEV, requires_grad=True)
    y = mod(x)
    assert y.shape == (2, 32, 32, 32)
    y.sum().backward()
    assert x.grad is not None and torch.isfinite(x.grad).all()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in mod.parameters())


def test_narrow_output_is_a_real_channels_last_tensor():
    """heads * dim_v = 12 is padded to 16 inside the layer: the output is its own allocation, so an in-place op after the
    layer works and the gradient still flows."""
    torch.manual_seed(0)
    mod = hb.nn.LambdaLayer(16, 12, 8, r=3).to(DEV)
    x = torch.randn(2, 16, 9, 7, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    y = mod(x)
    assert y.shape == (2, 12, 9, 7) and y.is_contiguous(memory_format=torch.channels_last) and y._base is None
    ref = y.detach().float().relu()
    y.relu_()
    assert torch.equal(y.detach().float(), ref)
    y.float().sum().backward()
    assert x.grad is not None and torch.isfinite(x.grad).all()


def test_bf16_channels_last_in_and_out():
    torch.manual_seed(0)
    mod = hb.nn.LambdaLayer(64, 64, 16, r=7).to(DEV)
    x = torch.randn(2, 64, 14, 14, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    y = mod(x)
    assert y.dtype == torch.bfloat16 and y.is_contiguous(memory_format=torch.channels_last)


def _run(mod, x, w):
    mod.zero_grad(set_to_none=True)
    x.grad = None
    y = mod(x)
    (y * w).sum().backward()
    return [y.detach().clone(), x.grad.clone()] + [p.grad.clone() for p in mod.parameters()]


@pytest.mark.parametrize("cfg", [(32, 64, 16, None, 7, 4, 1), (32, 48, 8, None, 5, 2, 4), (32, 32, 16, 64, None, 4, 2)])
def test_deterministic_and_graph_replay(cfg):
    c, o, dk, n, r, heads, u = cfg
    torch.manual_seed(0)
    mod = hb.nn.LambdaLayer(c, o, dk, n=n, r=r, num_heads=heads, dim_u=u).to(DEV)
    x = torch.randn(4, c, 8, 8, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    w = torch.randn(4, o, 8, 8, device=DEV).bfloat16()
    state = {k: v.clone() for k, v in mod.state_dict().items()}
    first = _run(mod, x, w)
    mod.load_state_dict(state)
    second = _run(mod, x, w)
    for a, b in zip(first, second):
        assert torch.equal(a, b)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _run(mod, x, w)
    torch.cuda.current_stream().wait_stream(side)
    mod.load_state_dict(state)
    mod.zero_grad(set_to_none=True)
    x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = mod(x)
        (y * w).sum().backward()
    mod.load_state_dict(state)
    graph.replay()
    torch.cuda.synchronize()
    replayed = [y, x.grad] + [p_.grad for p_ in mod.parameters()]
    for a, b in zip(first, replayed):
        assert torch.equal(a, b)


def _peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def test_peak_memory_below_eager():
    """Forward + backward of a LambdaResNet-sized layer (128 channels at 28², r = 23, batch 16) against the eager
    formulation (conv3d position lambda, in bf16) on the same parameters."""
    torch.manual_seed(0)
    mod = hb.nn.LambdaLayer(128, 128, 16, r=23).to(DEV)
    x = torch.randn(16, 128, 28, 28, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    x.requires_grad_(True)

    def ours():
        mod(x).float().sum().backward()

    def eager():
        y = O.lambda_module(x, mod, training=True, dtype=torch.bfloat16, core=O.lambda_core_conv3d)
        y.float().sum().backward()

    ours()
    eager()
    assert _peak(ours) < _peak(eager)
