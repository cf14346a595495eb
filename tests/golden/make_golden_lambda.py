"""Generates tests/golden/lambda_layer.pt by running the UNMODIFIED reference (frgfm/Holocron, a checkout named by the
HOLOCRON_REFERENCE environment variable) on seeded CPU inputs:

    HOLOCRON_REFERENCE=/path/to/Holocron python tests/golden/make_golden_lambda.py

It covers LambdaLayer and reuses the helpers of make_golden.py (importing it loads the reference and generates nothing).
"""
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from make_golden import OUT, describe_signature, holocron  # noqa: E402

# (in_channels, out_channels, dim_k, n, r, num_heads, dim_u) and the input shape; the first row is the reference's own
# test_lambdalayer layer and input, the others use H != W grids
CONFIGS = [
    ((8, 32, 16, None, 13, 4, 1), (2, 8, 32, 32)),
    ((8, 16, 8, None, 1, 2, 1), (2, 8, 6, 10)),
    ((8, 16, 16, None, 3, 1, 1), (2, 8, 6, 10)),
    ((8, 16, 8, None, 23, 4, 1), (2, 8, 5, 7)),       # the window is larger than the grid
    ((8, 24, 8, None, 5, 2, 4), (2, 8, 6, 10)),       # dim_u = 4, dim_v = 12
    ((3, 16, 8, None, 3, 4, 1), (2, 3, 6, 10)),       # in_channels = 3
    ((8, 16, 8, 20, None, 4, 2), (2, 8, 4, 5)),       # global variant, n = H * W
]


def _module(cfg):
    c, o, dk, n, r, heads, u = cfg
    return holocron.nn.LambdaLayer(c, o, dk, n=n, r=r, num_heads=heads, dim_u=u)


def gen_lambda():
    """LambdaLayer -> tests/golden/lambda_layer.pt: per configuration the seeded init, the input, the training-mode
    output, the gradients of the input and of every parameter for loss = sum(y * w) (w drawn from ``w_seed``), the
    running statistics after that forward, and the eval-mode output on the first sample; the signature, repr strings,
    state_dict layout, and the constructions and inputs the reference refuses."""
    d = {"signature": describe_signature(holocron.nn.LambdaLayer), "cases": []}
    for idx, (cfg, shape) in enumerate(CONFIGS):
        torch.manual_seed(300 + idx)
        mod = _module(cfg)
        init = {k: v.clone() for k, v in mod.state_dict().items()}
        x = torch.randn(*shape)
        xg = x.clone().requires_grad_(True)
        y = mod(xg)
        torch.manual_seed(900 + idx)
        wy = torch.randn(y.shape)   # not randn_like: the reference's output is a permuted view, w is drawn contiguous
        (y * wy).sum().backward()
        running = {k: v.clone() for k, v in mod.state_dict().items() if "running" in k or "num_batches" in k}
        mod.eval()
        with torch.no_grad():
            y_eval = mod(x[:1])
        d["cases"].append({
            "cfg": cfg, "shape": shape, "seed": 300 + idx, "w_seed": 900 + idx, "init": init, "x": x,
            "y": y.detach().clone(), "dx": xg.grad.clone(),
            "grads": {k: p.grad.clone() for k, p in mod.named_parameters()},
            "running": running, "y_eval": y_eval.clone(),
            "repr": repr(mod), "state_dict": [(k, tuple(v.shape)) for k, v in mod.state_dict().items()],
        })
    refused = []
    for kwargs in ({"in_channels": 8, "out_channels": 30, "dim_k": 16, "r": 3},
                   {"in_channels": 8, "out_channels": 32, "dim_k": 16, "r": 4},
                   {"in_channels": 8, "out_channels": 32, "dim_k": 16}):
        try:
            holocron.nn.LambdaLayer(**kwargs)
            raised, msg = None, None
        except AssertionError as e:
            raised, msg = type(e).__name__, str(e)
        refused.append({"kwargs": kwargs, "raised": raised, "message": msg})
    d["refused_constructions"] = refused
    errors = []
    for cfg, shape in (((8, 16, 8, 20, None, 4, 2), (1, 8, 4, 6)), ((8, 16, 8, 20, None, 4, 2), (1, 8, 5, 5))):
        torch.manual_seed(0)
        try:
            _module(cfg)(torch.randn(*shape))
            raised = None
        except RuntimeError as e:
            raised = type(e).__name__
        errors.append({"cfg": cfg, "shape": shape, "raised": raised})
    d["errors"] = errors
    torch.save(d, OUT / "lambda_layer.pt")


if __name__ == "__main__":
    gen_lambda()
    print("lambda_layer.pt", (OUT / "lambda_layer.pt").stat().st_size)
