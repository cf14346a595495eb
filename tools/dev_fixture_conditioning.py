"""Dev tool (CPU, needs a reference checkout): conditioning of candidate zoo fixtures.

For a reference model and a candidate (batch, size, parameter treatment) prints the rel-L2 distance between the
reference's fp32 logits and the SAME reference module tree run under CPU bf16 autocast - the error any bf16 execution
makes on that fixture. Used to choose tests/golden/zoo.pt setups whose bf16 spread is well below the test tolerance.
"""
import sys
import time

import torch

sys.path.insert(0, ".")
from oracle import reference_loader

holocron = reference_loader.load()


def rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


def condition(m, mode):
    """Parameter treatments that make a random-init net behave like a trained one (applied identically in both impls)."""
    g = torch.Generator().manual_seed(1234)
    bns = [mod for mod in m.modules() if isinstance(mod, torch.nn.BatchNorm2d)]
    with torch.no_grad():
        for bn in bns:
            if "affine" in mode:
                bn.weight.copy_(torch.rand(bn.weight.shape, generator=g) * 0.5 + 0.75)
                bn.bias.copy_(torch.rand(bn.bias.shape, generator=g) * 0.4 - 0.2)
            if "stats" in mode:
                bn.running_mean.copy_(torch.rand(bn.running_mean.shape, generator=g) * 0.4 - 0.2)
                bn.running_var.copy_(torch.rand(bn.running_var.shape, generator=g) * 1.0 + 0.5)


def run(name, b, sz, mode, train=True):
    torch.manual_seed(0)
    m = getattr(holocron.models, name)(num_classes=10)
    condition(m, mode)
    m.train(train)
    torch.manual_seed(1)
    x = torch.rand(b, 3, sz, sz)
    if "norm" in mode:
        x = (x - 0.45) / 0.225
    with torch.no_grad():
        t0 = time.time()
        ref = m(x)
        t1 = time.time()
        sd = {k: v.clone() for k, v in m.state_dict().items()}
        m.load_state_dict(sd)
        with torch.autocast("cpu", dtype=torch.bfloat16):
            lo = m(x)
    return rel(lo, ref), t1 - t0


if __name__ == "__main__":
    names = sys.argv[1].split(",")
    for name in names:
        for (b, sz) in [(2, 64), (8, 64), (8, 128)]:
            for mode in sys.argv[2].split(","):
                for train in (True, False):
                    e, t = run(name, b, sz, mode, train)
                    print(f"{name} b{b} {sz}x{sz} mode={mode} train={train}: autocast rel-L2 {e:.4f}  ({t:.1f}s fp32 fwd)", flush=True)
