"""Generates tests/golden/involution.pt by running the UNMODIFIED reference (frgfm/Holocron, a checkout named by the
HOLOCRON_REFERENCE environment variable) on seeded CPU inputs:

    HOLOCRON_REFERENCE=/path/to/Holocron python tests/golden/make_golden_involution.py

It covers Involution2d and reuses the helpers of make_golden.py (importing it loads the reference and generates nothing).
"""
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from make_golden import OUT, describe_signature, holocron  # noqa: E402

# (in_channels, kernel_size, padding, stride, dilation, groups, reduction_ratio); the first two rows are the reference's
# own test_involution2d
CONFIGS = [
    (8, 3, 1, 1, 1, 1, 2),
    (8, 3, 1, 2, 1, 1, 2),
    (16, 7, 3, 1, 1, 4, 4),
    (16, 3, 2, 1, 2, 2, 1),
    (24, 5, 2, 2, 1, 3, 3),
    (12, 3, 1, 1, 1, 6, 1.5),
    (32, 1, 0, 1, 1, 4, 2),
]
# input batch and grid: H != W catches a transposed index, both even so that the stride-2 rows have matching grids
SHAPE = (2, 8, 10)


def _module(cfg):
    c, k, p, s, d, g, r = cfg
    return holocron.nn.Involution2d(c, k, padding=p, stride=s, groups=g, dilation=d, reduction_ratio=r)


def gen_involution():
    """Involution2d -> tests/golden/involution.pt: per configuration the seeded init, the input, the output, and the
    gradients of the input and of the four parameters for loss = sum(y * w) with a random w; the signature, repr strings,
    state_dict layout, and the configurations the reference rejects with a RuntimeError."""
    d = {"configs": CONFIGS, "shape": SHAPE, "signature": describe_signature(holocron.nn.Involution2d), "cases": []}
    n, h, w = SHAPE
    for idx, cfg in enumerate(CONFIGS):
        torch.manual_seed(100 + idx)
        mod = _module(cfg)
        init = {k: v.clone() for k, v in mod.state_dict().items()}
        x = torch.randn(n, cfg[0], h, w)
        xg = x.clone().requires_grad_(True)
        y = mod(xg)
        wy = torch.randn_like(y)
        (y * wy).sum().backward()
        d["cases"].append({
            # clones: the reference's input gradient is a view into the larger buffer of its fold backward
            "cfg": cfg, "seed": 100 + idx, "init": init, "x": x, "y": y.detach().clone(), "w": wy,
            "dx": xg.grad.clone(),
            "grads": {k: p.grad.clone() for k, p in mod.named_parameters()},
            "repr": repr(mod), "state_dict": [(k, tuple(v.shape)) for k, v in mod.state_dict().items()],
        })
    errors = []
    # default padding=0 with K = 3 (6x6 unfold grid on an 8x8 input), an odd height with stride 2, C % G != 0
    for cfg, shape in (((8, 3, 0, 1, 1, 1, 1), (1, 8, 8, 8)), ((8, 3, 1, 2, 1, 1, 1), (1, 8, 9, 8)),
                       ((8, 3, 1, 1, 1, 3, 1), (1, 8, 8, 8))):
        torch.manual_seed(0)
        try:
            _module(cfg)(torch.randn(*shape))
            raised = None
        except RuntimeError as e:
            raised = type(e).__name__
        errors.append({"cfg": cfg, "shape": shape, "raised": raised})
    d["errors"] = errors
    torch.save(d, OUT / "involution.pt")


if __name__ == "__main__":
    gen_involution()
    print("involution.pt", (OUT / "involution.pt").stat().st_size)
