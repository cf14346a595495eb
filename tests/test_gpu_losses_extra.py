"""GPU tests of multilabel_cross_entropy, complement_cross_entropy and mutual_channel_loss (the fused kernels of
csrc/losses.cu): values and gradients against the reference's (tests/golden/losses_extra.pt), the reference's own loss
tests, low precision against the CPU restatements, full-size properties, captured training steps and the capture error
of the mutual channel loss."""
import pytest
import torch

import holocron_b200 as hb
from holocron_b200._lib import lib
from holocron_b200.models.classification.repvgg import RepVGG
from holocron_b200.nn import functional as F
from holocron_b200.nn._losses import mutual_channel_mask
from holocron_b200.trainer import TrainStep

import _losses_extra_oracle as O
from conftest import load_golden
from test_gpu_pointwise_losses_boxes import _loss_harness

pytestmark = pytest.mark.gpu

CE = torch.nn.functional.cross_entropy


def close(a, b, rtol, atol):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    torch.testing.assert_close(a, b, rtol=rtol, atol=atol, equal_nan=True)


def grad_of(fn, x):
    a = x.detach().clone().cuda().requires_grad_(True)
    y = fn(a)
    (gx,) = torch.autograd.grad(y.sum() if y.ndim else y, a)
    return y.detach(), gx


@pytest.fixture(scope="module")
def g():
    return load_golden("losses_extra")


def test_cross_entropies_vs_golden(g):
    for tag in ("cls", "seg"):
        x, t, w, soft = g[f"{tag}_x"], g[f"{tag}_t"].cuda(), g[f"{tag}_w"].cuda(), g[f"{tag}_soft"].cuda()
        for red in ("mean", "sum", "none"):
            for use_w in (False, True):
                wt = w if use_w else None
                for ii in (-100, 1):
                    key = f"{tag}_{red}_ii{ii}_w{int(use_w)}"
                    y, gx = grad_of(lambda a: F.multilabel_cross_entropy(a, soft, wt, ii, red), x)
                    close(y, g["mlce_" + key], 2e-5, 1e-6); close(gx, g["mlce_grad_" + key], 1e-4, 1e-6)
                    for gamma in (-1, 0.5, 0):
                        y, gx = grad_of(lambda a: F.complement_cross_entropy(a, t, wt, ii, red, gamma), x)
                        close(y, g[f"cce_g{gamma}_" + key], 2e-5, 1e-6)
                        close(gx, g[f"cce_g{gamma}_grad_" + key], 1e-4, 1e-6)
                key = f"{tag}_{red}_ii255_w{int(use_w)}"
                t255 = g[f"{tag}_t255"].cuda()
                y, gx = grad_of(lambda a: F.complement_cross_entropy(a, t255, wt, 255, red, 0), x)
                close(y, g["cce_g0_" + key], 2e-5, 1e-6); close(gx, g["cce_g0_grad_" + key], 1e-4, 1e-6)


def test_mutual_channel_loss_vs_golden(g):
    """Seeded as the reference was: the host draws the reference's masks, the kernels its values and gradients."""
    keys = [k[len("mcl_mask_"):] for k in g if k.startswith("mcl_mask_")]
    assert len(keys) == 2 * 2 * 3 * 2 * 2
    for key in keys:
        tag, xi, red, ii, w = key.split("_")
        base = f"mcl_{tag}_{xi}"
        wt = g[f"{base}_w"].cuda() if w == "w1" else None
        t = g[f"{base}_t"].cuda()
        torch.manual_seed(g["mcl_seed_" + key])
        y, gx = grad_of(lambda a: F.mutual_channel_loss(a, t, wt, int(ii[2:]), red, int(xi[2:])), g[f"{base}_x"])
        assert torch.equal(torch.get_rng_state(), g["mcl_rng_after_" + key]), key
        close(y, g["mcl_" + key], 2e-5, 1e-6); close(gx, g["mcl_grad_" + key], 1e-4, 1e-6)


def test_reference_loss_tests():
    """The reference's tests/test_nn_loss.py:70-133 on the CUDA path."""
    _loss_harness(F.multilabel_cross_entropy, multi_label=True)
    x = torch.rand(2, 4, 20, 20, device="cuda")
    target = torch.zeros_like(x)
    target[:, 0] = 1.0
    close(F.multilabel_cross_entropy(x, target), CE(x, target.argmax(dim=1)), 0, 1e-5)
    # complement CE: backprop with ignore_index = 0
    xg = torch.rand(2, 4, 20, 20, device="cuda", requires_grad=True)
    t = (4 * torch.rand(2, 20, 20, device="cuda")).long()
    F.complement_cross_entropy(xg, t, ignore_index=0).backward()
    assert torch.isfinite(xg.grad).all()
    # mutual channel loss behind a Linear layer, every reduction, then fp16 class weights through the module
    xi, num_classes = 2, 4
    x = torch.ones(2, xi * num_classes, device="cuda")
    x[:, 0] = 10
    target = torch.zeros(2, dtype=torch.long, device="cuda")
    mod = torch.nn.Linear(xi * num_classes, xi * num_classes).cuda()
    for reduction in ("mean", "sum", "none"):
        mod.zero_grad(set_to_none=True)
        loss = F.mutual_channel_loss(mod(x), target, ignore_index=0, reduction=reduction)
        if reduction == "none":
            assert loss.shape == (2,)
            loss = loss.sum()
        loss.backward()
        assert isinstance(mod.weight.grad, torch.Tensor)
    mod.zero_grad(set_to_none=True)
    criterion = hb.nn.MutualChannelLoss(weight=torch.ones(num_classes, dtype=torch.float16), ignore_index=0, xi=xi).cuda()
    criterion(mod(x), target).backward()
    assert isinstance(mod.weight.grad, torch.Tensor)
    assert repr(criterion) == f"MutualChannelLoss(reduction='mean', xi={xi}, alpha=1)"


def test_complement_gamma0_is_torch_cross_entropy():
    torch.manual_seed(3)
    for shape in ((64, 10), (4, 7, 9, 11), (16, 1000)):
        x = torch.randn(*shape, device="cuda", requires_grad=True)
        t = torch.randint(0, shape[1], (shape[0], *shape[2:]), device="cuda")
        t.view(-1)[::3] = 255
        w = torch.rand(shape[1], device="cuda") + 0.5
        for red in ("mean", "sum", "none"):
            for wt in (None, w):
                ours = F.complement_cross_entropy(x, t, wt, 255, red, 0)
                ref = CE(x, t, wt, ignore_index=255, reduction=red)
                close(ours, ref, 2e-5, 1e-6)
                go = torch.autograd.grad(ours.sum(), x)[0]
                gr = torch.autograd.grad(ref.sum(), x)[0]
                close(go, gr, 1e-4, 1e-6)


def test_mutual_channel_all_negative_logits():
    """Masked channels enter as 0 * x: with every logit negative each class logit is 0, the loss ln(cnum), no gradient."""
    x = -1 - torch.rand(4, 6, device="cuda")
    x.requires_grad_(True)
    t = torch.randint(0, 3, (4,), device="cuda")
    loss = F.mutual_channel_loss(x, t, alpha=0.0)
    close(loss, torch.tensor(3.0).log(), 1e-6, 0)
    loss.backward()
    assert torch.count_nonzero(x.grad) == 0


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_low_precision_vs_oracle(dtype):
    torch.manual_seed(5)
    x = (torch.randn(4, 12, 16, 16, device="cuda") * 2).to(dtype)
    t = torch.randint(0, 12, (4, 16, 16), device="cuda")
    soft = torch.softmax(torch.randn(4, 12, 16, 16, device="cuda"), 1).to(dtype)
    xf, sf = x.float().cpu(), soft.float().cpu()
    ulp = 2 ** -7
    y = F.multilabel_cross_entropy(x, soft, reduction="none")
    assert y.dtype == dtype
    close(y, O.multilabel_cross_entropy(xf, sf, reduction="none"), ulp, 1e-3)
    for gamma in (-1, 0.5):
        y = F.complement_cross_entropy(x, t, reduction="none", gamma=gamma)
        assert y.dtype == dtype
        close(y, O.complement_cross_entropy(xf, t.cpu(), reduction="none", gamma=gamma), ulp, 1e-3)
    tm = torch.randint(0, 4, (4, 16, 16), device="cuda")
    torch.manual_seed(6)
    y = F.mutual_channel_loss(x, tm, reduction="none", xi=3)
    torch.manual_seed(6)
    ref = O.mutual_channel_loss(xf, tm.cpu(), mutual_channel_mask(4, 3), reduction="none", xi=3)
    assert y.dtype == dtype
    close(y, ref, ulp, 1e-3)


def _properties(fn, x, ref_slice, seed=None):
    """sum == none.sum(), mean == none.mean(), a slice against the oracle, two calls (and two backwards) bit-identical."""
    def call(a, red):
        if seed is not None:
            torch.manual_seed(seed)
        return fn(a, red)
    rtol = 1e-4 if x.dtype == torch.float32 else 2 ** -7  # the reduced value is rounded to x.dtype
    none = call(x, "none")
    close(call(x, "sum"), none.float().sum(), rtol, 0)
    close(call(x, "mean"), none.float().mean(), rtol, 0)
    assert torch.equal(none, call(x, "none"))
    ref_slice(none)
    grads = []
    for _ in range(2):
        xr = x.detach().requires_grad_(True)
        grads.append(torch.autograd.grad(call(xr, "mean"), xr)[0])
    assert torch.equal(grads[0], grads[1])


def test_full_size_properties():
    torch.manual_seed(7)
    x = torch.randn(16, 21, 512, 512, device="cuda")
    t = torch.randint(0, 21, (16, 512, 512), device="cuda")
    _properties(lambda a, r: F.complement_cross_entropy(a, t, reduction=r), x,
                lambda none: close(none[:1, :64], O.complement_cross_entropy(x[:1, :, :64].cpu(), t[:1, :64].cpu(),
                                                                             reduction="none"), 1e-4, 1e-5))
    soft = torch.softmax(torch.randn_like(x), 1)
    _properties(lambda a, r: F.multilabel_cross_entropy(a, soft, reduction=r), x,
                lambda none: close(none[:1, :64], O.multilabel_cross_entropy(x[:1, :, :64].cpu(), soft[:1, :, :64].cpu(),
                                                                             reduction="none"), 1e-4, 1e-5))
    del x, t, soft
    xh = torch.randn(256, 1000, device="cuda")
    th = torch.randint(0, 1000, (256,), device="cuda")
    _properties(lambda a, r: F.complement_cross_entropy(a, th, reduction=r), xh,
                lambda none: close(none, O.complement_cross_entropy(xh.cpu(), th.cpu(), reduction="none"), 1e-4, 1e-5))
    xm = torch.randn(16, 63, 256, 256, device="cuda", dtype=torch.bfloat16)
    tm = torch.randint(0, 21, (16, 256, 256), device="cuda")
    torch.manual_seed(8)
    mask = mutual_channel_mask(21, 3)
    _properties(lambda a, r: F.mutual_channel_loss(a, tm, reduction=r, xi=3), xm,
                lambda none: close(none[:1], O.mutual_channel_loss(xm[:1].float().cpu(), tm[:1].cpu(), mask,
                                                                   reduction="none", xi=3), 2 ** -7, 1e-3), seed=8)


def _tiny():
    torch.manual_seed(0)
    return RepVGG([1, 1, 1], [16, 32, 64], 1, 1, num_classes=10)


def _batches(n, soft):
    gen = torch.Generator().manual_seed(41)
    out = []
    for _ in range(n):
        x = (torch.rand(8, 3, 32, 32, generator=gen) - 0.45) / 0.225
        t = torch.randint(0, 10, (8,), generator=gen)
        if soft:  # Mixup-style targets: lam * onehot(t) + (1 - lam) * onehot(t[perm])
            lam = 0.7
            oh = torch.nn.functional.one_hot(t, 10).float()
            t = lam * oh + (1 - lam) * oh[torch.randperm(8, generator=gen)]
        out.append((x, t))
    return out


@pytest.mark.parametrize("criterion", ["complement", "multilabel"])
def test_train_step_graph_matches_eager(criterion):
    """Every kernel on this path is deterministic: the captured step computes the same losses and parameters."""
    results = []
    for graph in (False, True):
        model = _tiny().cuda().to(memory_format=torch.channels_last).train()
        opt = hb.optim.AdaBelief(model.parameters(), lr=1e-3, betas=(0.95, 0.99), eps=1e-6, capturable=True)
        crit = hb.nn.ComplementCrossEntropy() if criterion == "complement" else hb.nn.MultiLabelCrossEntropy()
        step = TrainStep(model, crit, opt, graph=graph)
        losses = [step(x.cuda(), t.cuda()).float().clone() for x, t in _batches(5, criterion == "multilabel")]
        torch.cuda.synchronize()
        results.append((torch.stack(losses).cpu(), [p.detach().cpu().clone() for p in model.parameters()]))
    (l0, p0), (l1, p1) = results
    assert torch.isfinite(l0).all()
    assert torch.equal(l0, l1), (l0, l1)
    for a, b in zip(p0, p1):
        assert torch.equal(a, b)


def test_mutual_channel_loss_refuses_capture():
    x = torch.randn(2, 8, 5, 5, device="cuda")
    t = torch.randint(0, 4, (2, 5, 5), device="cuda")
    crit = hb.nn.MutualChannelLoss()
    graph = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    rng = torch.get_rng_state()
    launches = lib().hb_launch_count()
    with pytest.raises(RuntimeError, match="cannot run inside CUDA graph capture"):
        with torch.cuda.graph(graph):
            crit(x, t)
    assert lib().hb_launch_count() == launches
    assert torch.equal(torch.get_rng_state(), rng)
