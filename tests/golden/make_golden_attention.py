"""Generates tests/golden/attention.pt by running the UNMODIFIED reference (frgfm/Holocron, a checkout named by the
HOLOCRON_REFERENCE environment variable) on seeded CPU inputs:

    HOLOCRON_REFERENCE=/path/to/Holocron python tests/golden/make_golden_attention.py

It covers SAM, DimAttention and TripletAttention (holocron/nn/modules/attention.py) and conv_sequence's attention_layer
(holocron/models/utils.py), and reuses the helpers of make_golden.py (importing it loads the reference and generates
nothing).
"""
import sys
from pathlib import Path

import torch
from torch import nn

sys.path.insert(0, str(Path(__file__).resolve().parent))
from make_golden import OUT, describe_signature, holocron  # noqa: E402

ATT = holocron.nn.modules.attention
UTILS = holocron.models.utils


def _module_record(mod):
    return {"repr": repr(mod), "children": [(n, repr(m)) for n, m in mod.named_children()],
            "state_dict_layout": [(k, tuple(v.shape), str(v.dtype)) for k, v in mod.state_dict().items()]}


def _state(mod):
    return {k: v.detach().clone() for k, v in mod.state_dict().items()}


def _planted(shape, seed):
    """Small integers (ties along every dim), a NaN, and +-0.0 pairs on each reduced axis."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-3, 4, shape, generator=g).float()
    x[0, :, 1, 2] = 0.0          # channel axis: +-0.0 tie
    x[0, 1, 1, 2] = -0.0
    x[1, 2, :, 3] = -0.0         # H axis
    x[1, 2, 2, 3] = 0.0
    x[1, 3, 4, :] = 0.0          # W axis
    x[1, 3, 4, 0] = -0.0
    return x


def _step(mod, x, seed, training):
    mod.train(training)
    mod.zero_grad()
    xg = x.clone().requires_grad_(True)
    y = mod(xg)
    w = torch.randn(y.shape, generator=torch.Generator().manual_seed(seed)).to(y.dtype)
    (y * w).sum().backward()
    return {"training": training, "x": x, "w": w, "y": y.detach().clone(), "dx": xg.grad.clone(),
            "grads": {n: p.grad.clone() for n, p in mod.named_parameters()}}


def gen_attention():
    d = {"signatures": {name: describe_signature(getattr(ATT, name)) for name in ("SAM", "DimAttention",
                                                                                  "TripletAttention")},
         "all": list(ATT.__all__), "modules": [], "sam": [], "triplet": [], "dim": []}
    # construction records: seeded initialisation, repr, children, state_dict layout
    for ctor, args in (("SAM", (8,)), ("SAM", (3,)), ("DimAttention", (1,)), ("DimAttention", (2,)),
                       ("DimAttention", (3,)), ("TripletAttention", ())):
        torch.manual_seed(0)
        mod = getattr(ATT, ctor)(*args)
        d["modules"].append({"ctor": ctor, "args": args, **_module_record(mod), "state_dict": _state(mod)})

    seed = 100
    for c, dtype in ((8, torch.float32), (12, torch.float32), (3, torch.float32), (16, torch.bfloat16)):
        seed += 1
        torch.manual_seed(seed)
        mod = ATT.SAM(c).to(dtype)
        x = torch.randn(2, c, 5, 6).to(dtype)
        state = _state(mod)
        st = _step(mod, x, seed, True)
        d["sam"].append({"c": c, "state_dict": state, "x": x, "w": st["w"], "y": st["y"], "dx": st["dx"],
                         "dweight": st["grads"]["conv.weight"], "dbias": st["grads"]["conv.bias"]})

    # TripletAttention: two training steps then one evaluation step, on random and planted inputs
    for tag, shape in (("randn", (2, 6, 7, 5)), ("planted", (2, 5, 6, 7)), ("square", (3, 4, 4, 4))):
        seed += 1
        torch.manual_seed(seed)
        mod = ATT.TripletAttention()
        state = _state(mod)
        g = torch.Generator().manual_seed(seed)
        xs = [_planted(shape, seed + k) if tag == "planted" else torch.randn(shape, generator=g) for k in range(3)]
        steps = [_step(mod, xs[0], seed, True), _step(mod, xs[1], seed + 1, True), _step(mod, xs[2], seed + 2, False)]
        d["triplet"].append({"tag": tag, "state_dict": state, "steps": steps,
                             "buffers_after": {n: b.detach().clone() for n, b in mod.named_buffers()}})

    # DimAttention on its own, each dim, two training steps
    for dim in (1, 2, 3):
        seed += 1
        torch.manual_seed(seed)
        mod = ATT.DimAttention(dim)
        state = _state(mod)
        g = torch.Generator().manual_seed(seed)
        xs = [torch.randn(2, 6, 5, 7, generator=g) for _ in range(2)]
        steps = [_step(mod, xs[0], seed, True), _step(mod, xs[1], seed + 1, True)]
        d["dim"].append({"dim": dim, "state_dict": state, "steps": steps,
                         "buffers_after": {n: b.detach().clone() for n, b in mod.named_buffers()}})

    # planted NaN (evaluation mode: the NaN reaches its 7x7 plane neighbourhood only)
    seed += 1
    torch.manual_seed(seed)
    mod = ATT.TripletAttention()
    state = _state(mod)
    x = torch.randn(2, 5, 9, 8, generator=torch.Generator().manual_seed(seed))
    x[0, 1, 2, 3] = float("nan")
    d["nan"] = {"state_dict": state, "step": _step(mod, x, seed, False)}

    # conv_sequence with an attention layer: the layer list
    torch.manual_seed(0)
    layers = UTILS.conv_sequence(4, 8, nn.ReLU(inplace=True), nn.BatchNorm2d, kernel_size=3, padding=1,
                                 attention_layer=ATT.SAM)
    d["conv_sequence"] = [repr(m) for m in layers]
    torch.save(d, OUT / "attention.pt")


if __name__ == "__main__":
    gen_attention()
    print("attention.pt", (OUT / "attention.pt").stat().st_size)
