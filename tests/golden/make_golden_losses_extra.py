"""Generates tests/golden/losses_extra.pt by running the UNMODIFIED reference (frgfm/Holocron, a checkout named by the
HOLOCRON_REFERENCE environment variable) on seeded CPU inputs:

    HOLOCRON_REFERENCE=/path/to/Holocron python tests/golden/make_golden_losses_extra.py

It covers multilabel_cross_entropy, complement_cross_entropy, mutual_channel_loss and ClassBalancedWrapper, and reuses the
helpers of make_golden.py (importing it loads the reference and generates nothing).
"""
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from make_golden import OUT, describe_signature, grad_of, holocron  # noqa: E402

F = holocron.nn.functional


LOSSES_EXTRA = {"nn.functional": ["multilabel_cross_entropy", "complement_cross_entropy", "mutual_channel_loss"],
                "nn": ["MultiLabelCrossEntropy", "ComplementCrossEntropy", "ClassBalancedWrapper", "MutualChannelLoss"]}


def gen_losses_extra():
    """multilabel / complement cross entropy, mutual channel loss and ClassBalancedWrapper -> tests/golden/losses_extra.pt:
    seeded inputs, the reference's outputs and input gradients, the channel masks it drew, class-balanced weights, and the
    signatures and repr strings of the seven names."""
    import functools
    torch.manual_seed(13)
    d = {}
    for tag, shape in (("cls", (16, 10)), ("seg", (2, 5, 6, 7))):
        x = torch.randn(*shape) * 2
        k = shape[1]
        t = torch.randint(0, k, (shape[0],) + tuple(shape[2:]))
        t255 = t.clone()
        t255.view(-1)[::5] = 255
        w = torch.rand(k) + 0.5
        soft = torch.softmax(torch.randn(*shape), dim=1)
        d.update({f"{tag}_x": x, f"{tag}_t": t, f"{tag}_t255": t255, f"{tag}_w": w, f"{tag}_soft": soft})
        for red in ("mean", "sum", "none"):
            for use_w in (False, True):
                wt = w if use_w else None
                for ii in (-100, 1):
                    key = f"{tag}_{red}_ii{ii}_w{int(use_w)}"
                    y, (g,) = grad_of(lambda a: F.multilabel_cross_entropy(a, soft, wt, ii, red), x)
                    d["mlce_" + key], d["mlce_grad_" + key] = y, g
                    for gamma in (-1, 0.5, 0):
                        y, (g,) = grad_of(lambda a: F.complement_cross_entropy(a, t, wt, ii, red, gamma), x)
                        d[f"cce_g{gamma}_" + key], d[f"cce_g{gamma}_grad_" + key] = y, g
                # targets equal to ignore_index = 255: the reference accepts them only without the complement term
                key = f"{tag}_{red}_ii255_w{int(use_w)}"
                y, (g,) = grad_of(lambda a: F.complement_cross_entropy(a, t255, wt, 255, red, 0), x)
                d["cce_g0_" + key], d["cce_g0_grad_" + key] = y, g
    # mutual channel loss: (2, cnum*xi, 6, 7) and (16, cnum*xi); the masks are rebuilt from the reference's own randperm draws
    real_randperm = torch.randperm
    for tag, (n, cnum, spatial) in (("seg", (2, 5, (6, 7))), ("cls", (16, 10, ()))):
        for xi in (2, 3):
            x = torch.randn(n, cnum * xi, *spatial) * 2
            t = torch.randint(0, cnum, (n,) + tuple(spatial))
            w = torch.rand(cnum) + 0.5
            d.update({f"mcl_{tag}_xi{xi}_x": x, f"mcl_{tag}_xi{xi}_t": t, f"mcl_{tag}_xi{xi}_w": w})
            for red in ("mean", "sum", "none"):
                for ii in (-100, 1):
                    for use_w in (False, True):
                        key = f"mcl_{tag}_xi{xi}_{red}_ii{ii}_w{int(use_w)}"
                        seed = len(d)
                        draws = []

                        def recording_randperm(*a, **kw):
                            out = real_randperm(*a, **kw)
                            draws.append(out.clone())
                            return out

                        torch.manual_seed(seed)
                        torch.randperm = recording_randperm
                        try:
                            y, (g,) = grad_of(lambda a: F.mutual_channel_loss(a, t, w if use_w else None, ii, red, xi),
                                              x)
                        finally:
                            torch.randperm = real_randperm
                        base = torch.zeros(xi)
                        base[: (xi + 1) // 2] = 1
                        d[key], d[key.replace("mcl_", "mcl_grad_", 1)] = y, g
                        d[key.replace("mcl_", "mcl_mask_", 1)] = torch.stack([base[p] for p in draws])
                        d[key.replace("mcl_", "mcl_seed_", 1)] = seed
                        d[key.replace("mcl_", "mcl_rng_after_", 1)] = torch.get_rng_state()
    # ClassBalancedWrapper around torch's cross entropy, with and without an existing weight
    num_samples = torch.tensor([10, 50, 3, 200])
    for beta in (0.99, 0.9):
        crit = holocron.nn.ClassBalancedWrapper(torch.nn.CrossEntropyLoss(), num_samples, beta=beta)
        d[f"cb_beta{beta}_w0"] = crit.criterion.weight.clone()
        crit = holocron.nn.ClassBalancedWrapper(torch.nn.CrossEntropyLoss(weight=torch.tensor([1.0, 2.0, 0.5, 3.0])),
                                                num_samples, beta=beta)
        d[f"cb_beta{beta}_w1"] = crit.criterion.weight.clone()
        d[f"cb_beta{beta}_repr"] = repr(crit)
    d["cb_num_samples"] = num_samples
    sigs = {}
    for mod_path, names in LOSSES_EXTRA.items():
        mod = functools.reduce(getattr, mod_path.split("."), holocron)
        for name in names:
            sigs[f"{mod_path}.{name}"] = describe_signature(getattr(mod, name))
    d["signatures"] = sigs
    nn_ = holocron.nn
    d["reprs"] = {
        "MultiLabelCrossEntropy()": repr(nn_.MultiLabelCrossEntropy()),
        "MultiLabelCrossEntropy(reduction='sum')": repr(nn_.MultiLabelCrossEntropy(reduction="sum")),
        "ComplementCrossEntropy()": repr(nn_.ComplementCrossEntropy()),
        "ComplementCrossEntropy(gamma=0.5, reduction='none')": repr(nn_.ComplementCrossEntropy(gamma=0.5, reduction="none")),
        "MutualChannelLoss()": repr(nn_.MutualChannelLoss()),
        "MutualChannelLoss(xi=3, alpha=0.5)": repr(nn_.MutualChannelLoss(xi=3, alpha=0.5)),
        "ClassBalancedWrapper(CrossEntropyLoss(), num_samples)": repr(nn_.ClassBalancedWrapper(torch.nn.CrossEntropyLoss(),
                                                                                              num_samples)),
        "ClassBalancedWrapper(FocalLoss(), num_samples, beta=0.9)": repr(nn_.ClassBalancedWrapper(nn_.FocalLoss(),
                                                                                                 num_samples, beta=0.9)),
    }
    torch.save(d, OUT / "losses_extra.pt")


if __name__ == "__main__":
    gen_losses_extra()
    print("losses_extra.pt", (OUT / "losses_extra.pt").stat().st_size)
