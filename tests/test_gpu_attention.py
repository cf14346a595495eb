"""SAM, DimAttention and TripletAttention on the H100: per element against an fp64 restatement on the same input
(tests/_attention_oracle.py) in bf16 and fp32, train and eval, forward, dx and every parameter gradient; max-index
routing on planted ties and NaNs; the running statistics; the reference's fixture (tests/golden/attention.pt) through
the public modules; determinism and CUDA-graph replay; SAM inside a conv_sequence block; a realistic size.

Bars: fp32 outputs within 1e-4 relative plus 1e-5 of the largest reference magnitude (fp32 accumulation over at most a
few thousand terms, DESIGN.md §4). bf16 outputs are rounded once from fp32: half an ulp (2^-8 relative) of the exact
value, one ulp (2^-7) when fp32 rounding tips a value over a rounding boundary, plus the same fp32 absolute term.
Parameter gradients are fp32 in both dtypes (bf16 x and dy are exact in fp32 and fp64), so they take the fp32 bar with
the absolute term raised to 1e-4 for the sums over whole planes."""
import pytest
import torch
from torch import nn

import holocron_b200 as hb
from holocron_b200.models._blocks import FusedSequential
from holocron_b200.models.utils import conv_sequence

import _attention_oracle as O
from conftest import load_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ATT = hb.nn.modules.attention
DTYPES = [torch.bfloat16, torch.float32]
REL = {torch.bfloat16: 2.0 ** -7, torch.float32: 1e-4}


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def _close(got, ref, what, rel, atol_frac=1e-5):
    got = got.detach().cpu().double()
    ref = ref.detach().cpu().double()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert torch.equal(got.isnan(), ref.isnan()), f"{what}: NaN pattern differs"
    got, ref = got.nan_to_num(), ref.nan_to_num()
    bound = rel * ref.abs() + atol_frac * ref.abs().max().clamp_min(1e-30)
    bad = (got - ref).abs() > bound
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} off, first at {i}: got {float(got[i]):.7g} "
                             f"ref {float(ref[i]):.7g}")


# ---------------------------------------------------------------------------------------------------------------------
# SAM against fp64


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp32"])
@pytest.mark.parametrize("c", [1, 3, 8, 12, 64, 256])
@pytest.mark.parametrize("shape", [(2, 5, 7), (3, 1, 9), (2, 6, 1)], ids=["5x7", "1x9", "6x1"])
def test_sam_vs_fp64(shape, c, dtype):
    n, h, w = shape
    torch.manual_seed(c * 7 + h)
    mod = ATT.SAM(c).to(DEV)
    x = _cl(torch.randn(n, c, h, w, device=DEV).to(dtype)).requires_grad_(True)
    y = mod(x)
    assert y.dtype == dtype and y.shape == x.shape
    dy = torch.randn(y.shape, device=DEV).to(dtype)
    y.backward(dy)
    x64 = x.detach().cpu().double().requires_grad_(True)
    w64 = mod.conv.weight.detach().cpu().double().requires_grad_(True)
    b64 = mod.conv.bias.detach().cpu().double().requires_grad_(True)
    ref = O.sam(x64, w64, b64)
    ref.backward(dy.cpu().double())
    _close(y, ref, "y", REL[dtype])
    _close(x.grad, x64.grad, "dx", REL[dtype])
    _close(mod.conv.weight.grad, w64.grad, "dw", 1e-4, 1e-4)
    _close(mod.conv.bias.grad, b64.grad, "db", 1e-4, 1e-4)


def test_sam_errors():
    mod = ATT.SAM(4).to(DEV)
    with pytest.raises(RuntimeError):
        mod(torch.randn(1, 3, 4, 4, device=DEV))
    with pytest.raises(NotImplementedError):
        mod(torch.randn(4, 4, 4, device=DEV))


# ---------------------------------------------------------------------------------------------------------------------
# TripletAttention / DimAttention against fp64


def _run_triplet(mod, x, dy, training):
    """Module and fp64 oracle on the same input: returns ((y, dx, grads), (ref, dref, ref grads), ref params)."""
    mod.train(training)
    ps = {k: O.branch_params(getattr(mod, f"{k}_branch"), torch.float64, "cpu") for k in "chw"}
    xg = x.clone().requires_grad_(True)
    y = mod(xg)
    y.backward(dy)
    x64 = x.detach().cpu().double().requires_grad_(True)
    ref = O.triplet_attention(x64, ps, training)
    ref.backward(dy.cpu().double())
    return y, xg.grad, ref, x64.grad, ps


def _check_triplet(mod, x, dy, training, dtype):
    y, dx, ref, dref, ps = _run_triplet(mod, x, dy, training)
    assert y.dtype == dtype and y.shape == x.shape
    _close(y, ref, "y", REL[dtype])
    _close(dx, dref, "dx", REL[dtype])
    for k in "chw":
        br = getattr(mod, f"{k}_branch")
        conv, bn = br.compress[1], br.compress[2]
        _close(conv.weight.grad, ps[k]["conv_weight"].grad, f"{k}.conv.weight.grad", 1e-4, 1e-4)
        _close(bn.weight.grad, ps[k]["bn_weight"].grad, f"{k}.bn.weight.grad", 1e-4, 1e-4)
        _close(bn.bias.grad, ps[k]["bn_bias"].grad, f"{k}.bn.bias.grad", 1e-4, 1e-4)
        _close(bn.running_mean, ps[k]["running_mean"], f"{k}.running_mean", 1e-5, 1e-6)
        _close(bn.running_var, ps[k]["running_var"], f"{k}.running_var", 1e-5, 1e-6)


def _seeded_triplet(seed):
    torch.manual_seed(seed)
    mod = ATT.TripletAttention().to(DEV)
    with torch.no_grad():   # non-trivial affine parameters and running statistics
        for k in "chw":
            bn = getattr(mod, f"{k}_branch").compress[2]
            bn.weight.uniform_(0.5, 1.5)
            bn.bias.uniform_(-0.5, 0.5)
            bn.running_mean.uniform_(-0.5, 0.5)
            bn.running_var.uniform_(0.5, 2.0)
    return mod


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp32"])
@pytest.mark.parametrize("c", [1, 3, 8, 12, 64, 256])
def test_triplet_vs_fp64(c, dtype, training):
    mod = _seeded_triplet(c)
    x = _cl(torch.randn(2, c, 5, 7, device=DEV).to(dtype))
    dy = _cl(torch.randn(x.shape, device=DEV).to(dtype))
    _check_triplet(mod, x, dy, training, dtype)


# H != W, sides of 1, and H spanning several row blocks of the pool pass (bf16 C=256: 8 rows per block, fp32 C=256:
# 8, C=300: 6 or 4)
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp32"])
@pytest.mark.parametrize("shape", [(2, 16, 1, 9), (2, 16, 9, 1), (1, 256, 20, 6), (2, 300, 13, 5), (3, 64, 33, 2),
                                   (2, 24, 3, 40)],
                         ids=["h1", "w1", "hblocks256", "hblocks300", "tall", "wide"])
def test_triplet_shapes_vs_fp64(shape, dtype):
    mod = _seeded_triplet(sum(shape))
    x = _cl(torch.randn(shape, device=DEV).to(dtype))
    dy = _cl(torch.randn(shape, device=DEV).to(dtype))
    _check_triplet(mod, x, dy, True, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp32"])
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_triplet_ties_route_like_max_indices(dtype, training):
    """Small integers: ties along every reduced axis, so dx is right only where the gradient of each max goes to the
    element max(dim).indices names (the first one), as in the oracle."""
    g = torch.Generator().manual_seed(5)
    x = _cl(torch.randint(-2, 3, (2, 12, 9, 10), generator=g).float().to(dtype).to(DEV))
    x[0, :, 4, 4] = 0.0
    x[0, 3, 4, 4] = -0.0
    dy = _cl(torch.randn(x.shape, generator=g).to(dtype).to(DEV))
    _check_triplet(_seeded_triplet(9), x, dy, training, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp32"])
def test_triplet_nans_like_the_reference(dtype):
    """NaNs win the max (torch's rule): in eval mode they reach the 7x7 neighbourhood of their plane positions only, so
    the NaN pattern of y and dx checks where every plane routed them."""
    g = torch.Generator().manual_seed(6)
    x = torch.randn(2, 16, 12, 11, generator=g)
    x[0, 2, 1, 3] = float("nan")
    x[1, 9, 10, 0] = float("nan")
    x = _cl(x.to(dtype).to(DEV))
    dy = _cl(torch.randn(x.shape, generator=g).to(dtype).to(DEV))
    mod = _seeded_triplet(3).eval()
    y, dx, ref, dref, _ = _run_triplet(mod, x, dy, False)
    _close(y, ref, "y", REL[dtype])
    _close(dx, dref, "dx", REL[dtype])


@pytest.mark.parametrize("dim", [1, 2, 3, -1])
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp32"])
def test_dim_attention_alone(dim, dtype):
    torch.manual_seed(dim + 10)
    mod = ATT.DimAttention(dim).to(DEV)
    x = _cl(torch.randn(2, 12, 6, 9, device=DEV).to(dtype)).requires_grad_(True)
    p = O.branch_params(mod, torch.float64, "cpu")
    for _ in range(2):   # two training steps: the running statistics move twice
        x.grad = None
        y = mod(x)
        dy = torch.randn(y.shape, device=DEV).to(dtype)
        y.backward(dy)
        x64 = x.detach().cpu().double().requires_grad_(True)
        ref = O.dim_attention(x64, dim % 4, p, True)
        ref.backward(dy.cpu().double())
        _close(y, ref, "y", REL[dtype])
        _close(x.grad, x64.grad, "dx", REL[dtype])
    bn = mod.compress[2]
    _close(bn.running_mean, p["running_mean"], "running_mean", 1e-5, 1e-6)
    _close(bn.running_var, p["running_var"], "running_var", 1e-5, 1e-6)
    assert int(bn.num_batches_tracked) == 2


def test_triplet_errors():
    mod = ATT.TripletAttention().to(DEV)
    with pytest.raises(ValueError):   # one value per BatchNorm channel in the C branch's plane (N = H = W = 1)
        mod(torch.randn(1, 4, 1, 1, device=DEV))
    with pytest.raises(NotImplementedError):
        mod(torch.randn(4, 4, 4, device=DEV))
    mod.eval()
    assert mod(torch.randn(1, 4, 1, 1, device=DEV)).shape == (1, 4, 1, 1)


# ---------------------------------------------------------------------------------------------------------------------
# the reference's fixture through the public modules


def _load_state(mod, rec):
    mod.load_state_dict({k: v.to(DEV) for k, v in rec["state_dict"].items()})


def test_fixture_sam():
    d = load_golden("attention")
    for case in d["sam"]:
        mod = ATT.SAM(case["c"]).to(DEV)
        _load_state(mod, case)
        x = case["x"].to(DEV).requires_grad_(True)
        y = mod(x)
        (y * case["w"].to(DEV)).sum().backward()
        # in bf16 the reference rounds the convolution output, the gate and the product (and, backward, each partial
        # product) to bf16: a few ulps of 2^-7 between it and one rounding from fp32
        rel = REL[x.dtype] if x.dtype == torch.float32 else 2.0 ** -4
        _close(y, case["y"], "y", rel)
        # dx = dy g + ds w cancels; each term was rounded to bf16 there, so the bar adds 2^-6 of the largest |dx|
        _close(x.grad, case["dx"], "dx", rel, 1e-3 if x.dtype == torch.float32 else 2.0 ** -6)
        _close(mod.conv.weight.grad, case["dweight"], "dweight", 1e-4 if x.dtype == torch.float32 else 5e-2, 1e-2)
        _close(mod.conv.bias.grad, case["dbias"], "dbias", 1e-4 if x.dtype == torch.float32 else 5e-2, 1e-2)


def _fixture_cases():
    d = load_golden("attention")
    return ([(c["tag"], ATT.TripletAttention, c) for c in d["triplet"]]
            + [(f"dim{c['dim']}", lambda c=c: ATT.DimAttention(c["dim"]), c) for c in d["dim"]]
            + [("nan", ATT.TripletAttention, {"tag": "nan", "state_dict": d["nan"]["state_dict"],
                                             "steps": [d["nan"]["step"]]})])


def test_fixture_triplet_two_steps():
    """Train then eval, as the fixture recorded them: outputs, gradients, and the running statistics and
    num_batches_tracked of all three BatchNorms after two training steps; DimAttention alone for each dim; a planted
    NaN in eval mode."""
    for tag, ctor, case in _fixture_cases():
        mod = ctor().to(DEV)
        _load_state(mod, case)
        for step in case["steps"]:
            mod.train(step["training"])
            mod.zero_grad()
            x = step["x"].to(DEV).requires_grad_(True)
            y = mod(x)
            (y * step["w"].to(DEV)).sum().backward()
            _close(y, step["y"], f"{tag} y", 1e-4, 1e-4)
            _close(x.grad, step["dx"], f"{tag} dx", 1e-4, 1e-4)
            for name, p in mod.named_parameters():
                _close(p.grad, step["grads"][name], f"{tag} {name}.grad", 1e-3, 1e-3)
        for name, b in mod.named_buffers():
            if "buffers_after" not in case:
                break
            ref = case["buffers_after"][name]
            if name.endswith("num_batches_tracked"):
                assert int(b) == int(ref), name
            else:
                _close(b, ref, name, 1e-5, 1e-6)


# ---------------------------------------------------------------------------------------------------------------------
# determinism, graphs, models, size


def _triplet_step(mod, x, dy):
    mod.zero_grad(set_to_none=False)
    xg = x.clone().requires_grad_(True)
    y = mod(xg)
    y.backward(dy)
    return [y.detach().clone(), xg.grad.clone()] + [p.grad.clone() for p in mod.parameters()]


@pytest.mark.parametrize("layer", ["sam", "triplet"])
def test_deterministic_and_graph_replay(layer):
    torch.manual_seed(0)
    mod = (ATT.SAM(64) if layer == "sam" else _seeded_triplet(0)).to(DEV).train()
    x = _cl(torch.randn(4, 64, 28, 28, device=DEV).to(torch.bfloat16))
    dy = _cl(torch.randn(x.shape, device=DEV).to(torch.bfloat16))
    state = {k: v.clone() for k, v in mod.state_dict().items()}
    a = _triplet_step(mod, x, dy)
    mod.load_state_dict(state)
    b = _triplet_step(mod, x, dy)
    b_bufs = {k: v.clone() for k, v in mod.named_buffers()}
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    # capture one step (after a warm-up on a side stream), replay, compare with eager
    mod.load_state_dict(state)
    xs = x.clone().requires_grad_(True)
    for p in mod.parameters():
        p.grad = torch.zeros_like(p)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            mod.load_state_dict(state)
            xs.grad = None
            mod(xs).backward(dy)
    torch.cuda.current_stream().wait_stream(s)
    mod.load_state_dict(state)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for p in mod.parameters():
            p.grad.zero_()
        y = mod(xs)
        y.backward(dy)
    mod.load_state_dict(state)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(y, a[0])
    for p, ref in zip(mod.parameters(), a[2:]):
        assert torch.equal(p.grad, ref)
    if layer == "triplet":   # the captured step updated the running statistics as the eager one did
        for name, buf in mod.named_buffers():
            assert torch.equal(buf, b_bufs[name]), name


def test_sam_inside_conv_sequence():
    torch.manual_seed(1)
    layers = conv_sequence(16, 32, nn.ReLU(inplace=True), nn.BatchNorm2d, kernel_size=3, padding=1,
                           attention_layer=ATT.SAM)
    assert isinstance(layers[-1], ATT.SAM) and layers[-1].conv.in_channels == 32
    seq = FusedSequential(*layers).to(DEV).train()
    head = FusedSequential(*layers[:-1])
    x = _cl(torch.randn(4, 16, 20, 20, device=DEV).to(torch.bfloat16)).requires_grad_(True)
    y = seq(x)
    assert y.dtype == torch.bfloat16 and torch.isfinite(y).all()
    u = head(x).detach()
    assert u.is_contiguous(memory_format=torch.channels_last)
    u64 = u.cpu().double()
    ref = O.sam(u64, layers[-1].conv.weight.detach().cpu().double(), layers[-1].conv.bias.detach().cpu().double())
    _close(layers[-1](u), ref, "sam(conv output)", REL[torch.bfloat16])
    y.float().square().sum().backward()
    assert torch.isfinite(x.grad).all() and torch.isfinite(layers[-1].conv.weight.grad).all()


@pytest.mark.parametrize("layer", ["sam", "triplet"])
def test_realistic_size(layer):
    """N=32, C=256, 56x56 in bf16 (a ResNet-50 stage-1 output), training mode."""
    torch.manual_seed(2)
    x = _cl(torch.randn(32, 256, 56, 56, device=DEV).to(torch.bfloat16))
    dy = _cl(torch.randn(x.shape, device=DEV).to(torch.bfloat16))
    if layer == "sam":
        mod = ATT.SAM(256).to(DEV)
        xg = x.clone().requires_grad_(True)
        y = mod(xg)
        y.backward(dy)
        x64 = x.cpu().double().requires_grad_(True)
        w64 = mod.conv.weight.detach().cpu().double().requires_grad_(True)
        b64 = mod.conv.bias.detach().cpu().double().requires_grad_(True)
        ref = O.sam(x64, w64, b64)
        ref.backward(dy.cpu().double())
        _close(y, ref, "y", REL[torch.bfloat16])
        _close(xg.grad, x64.grad, "dx", REL[torch.bfloat16])
        _close(mod.conv.weight.grad, w64.grad, "dw", 1e-4, 1e-4)
    else:
        _check_triplet(_seeded_triplet(2), x, dy, True, torch.bfloat16)
