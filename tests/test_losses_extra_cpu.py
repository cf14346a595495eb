"""CPU checks of the multilabel / complement cross entropy, mutual channel loss and ClassBalancedWrapper surface against
tests/golden/losses_extra.pt (written by make_golden_losses_extra.py from the unmodified reference): the CPU restatements
against the reference's values and gradients, the signatures and repr strings, the class-balanced weights, the shape error
and the host-side channel-mask draw."""
import inspect

import pytest
import torch

import holocron_b200 as hb
from holocron_b200.nn._losses import mutual_channel_mask

import _losses_extra_oracle as O
from conftest import load_golden


@pytest.fixture(scope="module")
def g():
    return load_golden("losses_extra")


def grad_of(fn, x):
    a = x.clone().requires_grad_(True)
    y = fn(a)
    (gx,) = torch.autograd.grad(y.sum() if y.ndim else y, a)
    return y.detach(), gx


def close(a, b, rtol=1e-6, atol=1e-7):
    assert a.shape == b.shape, (a.shape, b.shape)
    torch.testing.assert_close(a, b, rtol=rtol, atol=atol)


def test_oracle_cross_entropies_vs_golden(g):
    for tag in ("cls", "seg"):
        x, t, w, soft = g[f"{tag}_x"], g[f"{tag}_t"], g[f"{tag}_w"], g[f"{tag}_soft"]
        for red in ("mean", "sum", "none"):
            for use_w in (False, True):
                wt = w if use_w else None
                for ii in (-100, 1):
                    key = f"{tag}_{red}_ii{ii}_w{int(use_w)}"
                    y, gx = grad_of(lambda a: O.multilabel_cross_entropy(a, soft, wt, ii, red), x)
                    close(y, g["mlce_" + key]); close(gx, g["mlce_grad_" + key])
                    for gamma in (-1, 0.5, 0):
                        y, gx = grad_of(lambda a: O.complement_cross_entropy(a, t, wt, ii, red, gamma), x)
                        close(y, g[f"cce_g{gamma}_" + key]); close(gx, g[f"cce_g{gamma}_grad_" + key])
                key = f"{tag}_{red}_ii255_w{int(use_w)}"
                y, gx = grad_of(lambda a: O.complement_cross_entropy(a, g[f"{tag}_t255"], wt, 255, red, 0), x)
                close(y, g["cce_g0_" + key]); close(gx, g["cce_g0_grad_" + key])


def _mcl_keys(g):
    return [k for k in g if k.startswith("mcl_mask_")]


def test_oracle_mutual_channel_vs_golden(g):
    keys = _mcl_keys(g)
    assert len(keys) == 2 * 2 * 3 * 2 * 2
    for mk in keys:
        tag, xi, red, ii, w = mk[len("mcl_mask_"):].split("_")
        base = f"mcl_{tag}_{xi}"
        wt = g[f"{base}_w"] if w == "w1" else None
        y, gx = grad_of(lambda a: O.mutual_channel_loss(a, g[f"{base}_t"], g[mk], wt, int(ii[2:]), red, int(xi[2:])),
                        g[f"{base}_x"])
        key = mk.replace("mcl_mask_", "")
        close(y, g["mcl_" + key]); close(gx, g["mcl_grad_" + key])


def test_mask_draw_reproduces_the_reference(g):
    for mk in _mcl_keys(g):
        key = mk.replace("mcl_mask_", "")
        cnum, xi = g[mk].shape
        torch.manual_seed(g["mcl_seed_" + key])
        mask = mutual_channel_mask(cnum, xi)
        assert torch.equal(mask, g[mk]), key
        assert torch.equal(torch.get_rng_state(), g["mcl_rng_after_" + key]), key


def _describe(obj):
    target = obj.__init__ if inspect.isclass(obj) else obj
    out = []
    for name, p in inspect.signature(target).parameters.items():
        if name == "self":
            continue
        out.append([name, p.kind.name, None if p.default is inspect.Parameter.empty else repr(p.default)])
    return out


def test_signatures_and_reprs_match_the_reference(g):
    for path, ref in g["signatures"].items():
        mod_path, name = path.rsplit(".", 1)
        mod = hb.nn.functional if mod_path == "nn.functional" else hb.nn
        assert _describe(getattr(mod, name)) == ref, path
    assert {"multilabel_cross_entropy", "complement_cross_entropy", "mutual_channel_loss"} <= set(hb.nn.functional.__all__)
    num_samples = g["cb_num_samples"]
    ours = {
        "MultiLabelCrossEntropy()": hb.nn.MultiLabelCrossEntropy(),
        "MultiLabelCrossEntropy(reduction='sum')": hb.nn.MultiLabelCrossEntropy(reduction="sum"),
        "ComplementCrossEntropy()": hb.nn.ComplementCrossEntropy(),
        "ComplementCrossEntropy(gamma=0.5, reduction='none')": hb.nn.ComplementCrossEntropy(gamma=0.5, reduction="none"),
        "MutualChannelLoss()": hb.nn.MutualChannelLoss(),
        "MutualChannelLoss(xi=3, alpha=0.5)": hb.nn.MutualChannelLoss(xi=3, alpha=0.5),
        "ClassBalancedWrapper(CrossEntropyLoss(), num_samples)": hb.nn.ClassBalancedWrapper(torch.nn.CrossEntropyLoss(),
                                                                                            num_samples),
        "ClassBalancedWrapper(FocalLoss(), num_samples, beta=0.9)": hb.nn.ClassBalancedWrapper(hb.nn.FocalLoss(),
                                                                                               num_samples, beta=0.9),
    }
    assert set(ours) == set(g["reprs"])
    for k, m in ours.items():
        assert repr(m) == g["reprs"][k], k


def test_class_balanced_wrapper_around_torch_cross_entropy(g):
    num_samples = g["cb_num_samples"]
    for beta in (0.99, 0.9):
        crit = hb.nn.ClassBalancedWrapper(torch.nn.CrossEntropyLoss(), num_samples, beta=beta)
        assert isinstance(crit.criterion, torch.nn.CrossEntropyLoss)
        close(crit.criterion.weight, g[f"cb_beta{beta}_w0"], 0, 0)
        base = torch.nn.CrossEntropyLoss(weight=torch.tensor([1.0, 2.0, 0.5, 3.0]))
        existing = base.weight
        crit = hb.nn.ClassBalancedWrapper(base, num_samples, beta=beta)
        assert crit.criterion.weight is existing  # multiplied in place
        close(crit.criterion.weight, g[f"cb_beta{beta}_w1"], 0, 0)
        assert repr(crit) == g[f"cb_beta{beta}_repr"]
        x, t = torch.randn(3, 4), torch.tensor([0, 3, 1])
        close(crit(x, t), torch.nn.functional.cross_entropy(x, t, g[f"cb_beta{beta}_w1"]), 0, 0)


def test_mutual_channel_channel_count_must_divide():
    # the reference's x.view(b, cnum, xi, -1) raises; nothing is drawn from the generator before that
    x, t = torch.randn(2, 5, 6, 7), torch.zeros(2, 6, 7, dtype=torch.long)
    state = torch.get_rng_state()
    with pytest.raises(RuntimeError, match="is invalid for input of size"):
        hb.nn.functional.mutual_channel_loss(x, t, xi=2)
    assert torch.equal(torch.get_rng_state(), state)


def test_cpu_tensors_are_rejected():
    x, t = torch.randn(4, 6), torch.zeros(4, dtype=torch.long)
    for fn, tgt in ((hb.nn.functional.multilabel_cross_entropy, torch.rand(4, 6)),
                    (hb.nn.functional.complement_cross_entropy, t), (hb.nn.functional.mutual_channel_loss, t)):
        with pytest.raises(hb.HolocronB200Error):
            fn(x, tgt)
