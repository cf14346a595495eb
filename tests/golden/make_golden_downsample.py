"""Generates tests/golden/downsample.pt by running the UNMODIFIED reference (frgfm/Holocron, a checkout named by the
HOLOCRON_REFERENCE environment variable) on seeded CPU inputs:

    HOLOCRON_REFERENCE=/path/to/Holocron python tests/golden/make_golden_downsample.py

It covers BlurPool2d, GlobalMaxPool2d, ZPool and z_pool, and reuses the helpers of make_golden.py (importing it loads the
reference and generates nothing).
"""
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from make_golden import OUT, describe_signature, holocron  # noqa: E402

DS = holocron.nn.modules.downsample
F = holocron.nn.functional

BLUR_KS = (2, 3, 4, 5, 7)
BLUR_STRIDES = (1, 2, 3)
Z_DIMS = (1, 2, 3, -1)


def _run(fn, x, seed):
    """(y, w, dx) of loss = sum(y * w) with a seeded w."""
    xg = x.clone().requires_grad_(True)
    y = fn(xg)
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(y.shape, generator=g).to(y.dtype)
    (y * w).sum().backward()
    return y.detach().clone(), w, xg.grad.clone()


def _module_record(mod):
    return {"repr": repr(mod), "children": [(n, repr(m)) for n, m in mod.named_children()],
            "state_dict": [(k, tuple(v.shape)) for k, v in mod.state_dict().items()]}


def _planted(shape, seed):
    """Small integer values (ties along every dim), one NaN pair, and +-0.0 pairs in otherwise negative rows."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-4, 4, shape, generator=g).float()
    x[0, 1, 2, 3] = float("nan")
    x[0, 1, 4, 1] = float("nan")
    x[1, 2] = -torch.rand(shape[2:], generator=g) - 1.0      # a row of the max over H*W that only +-0.0 decide
    x[1, 2, 0, 2] = 0.0
    x[1, 2, 3, 4] = -0.0
    x[1, 3] = -torch.rand(shape[2:], generator=g) - 1.0
    x[1, 3, 1, 1] = -0.0
    x[1, 3, 2, 5] = 0.0
    x[0, :, 5, 6] = 0.0                                       # a channel vector of zeros with one -0.0 (dim 1 tie)
    x[0, 0, 5, 6] = -0.0
    return x


def gen_downsample():
    d = {"signatures": {name: describe_signature(getattr(DS, name))
                        for name in ("BlurPool2d", "GlobalMaxPool2d", "ZPool")},
         "z_pool_signature": describe_signature(F.z_pool),
         "modules": [], "blur": [], "gmp": [], "zpool": [], "errors": []}
    for ctor, args in (("BlurPool2d", (4,)), ("BlurPool2d", (8, 5, 3)), ("BlurPool2d", (16, 8, 2)),
                       ("BlurPool2d", (3, 2, 1)), ("GlobalMaxPool2d", ()), ("GlobalMaxPool2d", (True,)),
                       ("ZPool", ()), ("ZPool", (2,))):
        mod = getattr(DS, ctor)(*args)
        rec = {"ctor": ctor, "args": args, **_module_record(mod)}
        if ctor == "BlurPool2d":
            rec["coeffs"] = mod._coeffs.clone()
            rec["filter_bf16"] = mod._create_filter(torch.empty(0, dtype=torch.bfloat16))[0, 0].clone()
            rec["filter_fp32"] = mod._create_filter(torch.empty(0))[0, 0].clone()
        d["modules"].append(rec)

    seed = 0
    for k in BLUR_KS:
        for s in BLUR_STRIDES:
            p = ((s - 1) + (k - 1)) // 2
            # H != W with odd sides, and the smallest legal side: p + 1 (every reflection path of the border), or k - 2p
            # where the padded side would be shorter than the filter
            side = max(p + 1, k - 2 * p)
            for shape in ((2, 3, 11, 8), (1, 2, side, side + 1)):
                for dtype in (torch.float32, torch.bfloat16):
                    seed += 1
                    torch.manual_seed(seed)
                    x = torch.randn(shape).to(dtype)
                    mod = DS.BlurPool2d(shape[1], k, s)
                    y, w, dx = _run(mod, x, seed)
                    d["blur"].append({"k": k, "s": s, "x": x, "w": w, "y": y, "dx": dx})

    for dtype in (torch.float32, torch.bfloat16):
        for tag, x in (("planted", _planted((2, 5, 6, 7), 3)), ("randn", torch.randn(2, 5, 6, 7, generator=torch.Generator().manual_seed(4)))):
            x = x.to(dtype)
            for flatten in (False, True):
                seed += 1
                y, w, dx = _run(DS.GlobalMaxPool2d(flatten), x, seed)
                d["gmp"].append({"tag": tag, "flatten": flatten, "x": x, "w": w, "y": y, "dx": dx})
            for dim in Z_DIMS:
                seed += 1
                y, w, dx = _run(lambda t: F.z_pool(t, dim), x, seed)
                d["zpool"].append({"tag": tag, "dim": dim, "x": x, "w": w, "y": y, "dx": dx})

    def _raised(fn):
        try:
            fn()
        except Exception as e:  # noqa: BLE001 - the exception type is what is recorded
            return type(e).__name__
        return None

    d["errors"] = [
        {"case": "kernel_size_1", "ctor": (4, 1, 2), "shape": None, "raised": _raised(lambda: DS.BlurPool2d(4, 1))},
        {"case": "kernel_size_0", "ctor": (1, 0, 2), "shape": None, "raised": _raised(lambda: DS.BlurPool2d(1, 0))},
        {"case": "channel_mismatch", "ctor": (4, 3, 2), "shape": (1, 3, 8, 8),
         "raised": _raised(lambda: DS.BlurPool2d(4, 3, 2)(torch.randn(1, 3, 8, 8)))},
        {"case": "pad_ge_height", "ctor": (2, 5, 3), "shape": (1, 2, 3, 9),
         "raised": _raised(lambda: DS.BlurPool2d(2, 5, 3)(torch.randn(1, 2, 3, 9)))},
        {"case": "pad_ge_width", "ctor": (2, 4, 2), "shape": (1, 2, 9, 2),
         "raised": _raised(lambda: DS.BlurPool2d(2, 4, 2)(torch.randn(1, 2, 9, 2)))},
        {"case": "padded_side_below_kernel", "ctor": (2, 2, 1), "shape": (1, 2, 1, 5),
         "raised": _raised(lambda: DS.BlurPool2d(2, 2, 1)(torch.randn(1, 2, 1, 5)))},
    ]
    torch.save(d, OUT / "downsample.pt")


if __name__ == "__main__":
    gen_downsample()
    print("downsample.pt", (OUT / "downsample.pt").stat().st_size)
