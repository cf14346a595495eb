"""Leaf-kernel micro rows of the hot path (BASELINE.md §3.3, `python bench.py --micro`): every bandwidth-bound kernel
north_star names, at the configurations' sizes, timed with CUDA events through the PUBLIC Python API (forward, and
forward+backward where the op is differentiable) and reported as achieved GB/s over the ALGORITHMIC bytes of SURVEY.md
§8(d) against the measured HBM copy peak. Inputs are larger than the L2 (50 MB on an H100) or the L2 is flushed between iterations
(a 256 MB scratch write), stated per row."""
import sys
from pathlib import Path

import torch
import torch.nn.functional as TF


def _time(fn, flush=None, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        # park the stream behind a ~10 ms spin kernel: the Python / autograd / table-building host work of the call then
        # overlaps the spin and the event pair brackets GPU time only (what the kernels cost inside a captured step)
        torch.cuda._sleep(int(2e7))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
    return tot / iters


def run_micro(peaks):
    import holocron_b200 as hb
    from holocron_b200.nn import functional as F
    from holocron_b200.nn._losses import mutual_channel_mask
    from holocron_b200.ops import boxes as B
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))
    import _losses_extra_oracle as OX
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, device=dev, dtype=torch.uint8)
    rows = []

    def row(name, shape, ms, byts, flops=None, l2="inputs > L2"):
        r = {"kernel": name, "shape": shape, "ms": round(ms, 4), "algorithmic_MB": round(byts / 1e6, 2),
             "GB/s": round(byts / ms / 1e6, 1), "frac_hbm": round(byts / ms / 1e6 / peaks["hbm_gbs"], 3), "l2": l2}
        if flops:
            r["TFLOP/s"] = round(flops / ms / 1e9, 2)
        rows.append(r)

    # ---- activations (Darknet-size tensor: 256 x 64 x 112 x 112 bf16 = 411 MB)
    x = torch.randn(256, 64, 112, 112, device=dev, dtype=torch.bfloat16)
    n = x.numel()
    for name, fn in (("hard_mish", F.hard_mish), ("nl_relu", F.nl_relu)):
        row(f"{name} fwd", list(x.shape), _time(lambda: fn(x)), 2 * 2 * n)
        xr = x.clone().requires_grad_(True)
        g = torch.randn_like(x)
        y = fn(xr)
        row(f"{name} bwd", list(x.shape), _time(lambda: torch.autograd.grad(y, xr, g, retain_graph=True)), 3 * 2 * n)
        del xr, y, g
    del x
    # ---- losses (segmentation logits 16 x 21 x 512 x 512 fp32 = 352 MB; dice 16 x 21 x 256 x 256)
    x = torch.randn(16, 21, 512, 512, device=dev)
    t = torch.randint(0, 21, (16, 512, 512), device=dev)
    nk, npos = x.numel(), t.numel()
    for name, fn in (("focal_loss", F.focal_loss), ("poly_loss", F.poly_loss)):
        row(f"{name} fwd", list(x.shape), _time(lambda: fn(x, t)), nk * 4 + npos * 8 + 4)
        xr = x.clone().requires_grad_(True)
        loss = fn(xr, t)
        row(f"{name} bwd", list(x.shape), _time(lambda: torch.autograd.grad(loss, xr, retain_graph=True)), 2 * nk * 4 + npos * 8)
        del xr, loss
    # complement and multi-label cross entropy on the same logits, each beside the CPU oracle's eager formulation run on
    # the same GPU (the `eager` rows: what the reference's torch code costs there)
    soft = torch.softmax(torch.randn_like(x), 1)
    for name, fn, tgt, fb, bb in (
            ("complement_cross_entropy", F.complement_cross_entropy, t, nk * 4 + npos * 8 + 4, 2 * nk * 4 + npos * 8),
            ("multilabel_cross_entropy", F.multilabel_cross_entropy, soft, 2 * nk * 4 + 4, 3 * nk * 4)):
        for impl, f in ((name, fn), (f"{name} eager", getattr(OX, name))):
            row(f"{impl} fwd", list(x.shape), _time(lambda: f(x, tgt)), fb)
            xr = x.clone().requires_grad_(True)
            loss = f(xr, tgt)
            row(f"{impl} bwd", list(x.shape), _time(lambda: torch.autograd.grad(loss, xr, retain_graph=True)), bb)
            del xr, loss
    del x, t, soft
    # ImageNet head: 256 x 1000 logits (1 MB, L2 flushed), one warp per row
    x = torch.randn(256, 1000, device=dev)
    t = torch.randint(0, 1000, (256,), device=dev)
    for impl, f in (("complement_cross_entropy", F.complement_cross_entropy),
                    ("complement_cross_entropy eager", OX.complement_cross_entropy)):
        row(f"{impl} fwd", list(x.shape), _time(lambda: f(x, t), flush), x.numel() * 4 + 256 * 8 + 4, l2="L2 flushed")
        xr = x.clone().requires_grad_(True)
        loss = f(xr, t)
        row(f"{impl} bwd", list(x.shape), _time(lambda: torch.autograd.grad(loss, xr, retain_graph=True), flush),
            2 * x.numel() * 4 + 256 * 8, l2="L2 flushed")
        del xr, loss
    del x, t
    # mutual channel loss: 16 x 63 x 256 x 256 bf16 (132 MB, xi = 3: 21 classes); algorithmic bytes = the features once
    # and the targets (forward), plus the feature gradient (backward)
    x = torch.randn(16, 63, 256, 256, device=dev, dtype=torch.bfloat16)
    t = torch.randint(0, 21, (16, 256, 256), device=dev)
    nk, npos = x.numel(), t.numel()
    mask = mutual_channel_mask(21, 3).to(dev)
    for impl, f in (("mutual_channel_loss", lambda a: F.mutual_channel_loss(a, t, xi=3)),
                    ("mutual_channel_loss eager", lambda a: OX.mutual_channel_loss(a, t, mask, xi=3))):
        row(f"{impl} fwd", list(x.shape), _time(lambda: f(x), flush), nk * 2 + npos * 8, l2="L2 flushed")
        xr = x.clone().requires_grad_(True)
        loss = f(xr)
        row(f"{impl} bwd", list(x.shape), _time(lambda: torch.autograd.grad(loss, xr, retain_graph=True), flush),
            2 * nk * 2 + npos * 8, l2="L2 flushed")
        del xr, loss
    del x, t
    x = torch.softmax(torch.randn(16, 21, 256, 256, device=dev), 1)
    oh = TF.one_hot(torch.randint(0, 21, (16, 256, 256), device=dev), 21).movedim(-1, 1).float().contiguous()
    row("dice_loss fwd", list(x.shape), _time(lambda: F.dice_loss(x, oh), flush), 2 * x.numel() * 4, l2="L2 flushed")
    xr = x.clone().requires_grad_(True)
    loss = F.dice_loss(xr, oh)
    row("dice_loss bwd", list(x.shape), _time(lambda: torch.autograd.grad(loss, xr, retain_graph=True), flush), 2 * x.numel() * 4,
        l2="L2 flushed")
    del x, oh, xr, loss
    # ---- pairwise box losses (4096 x 4096 -> 67 MB fp32 output)
    b1 = torch.rand(4096, 4, device=dev); b1[:, 2:] += b1[:, :2]
    b2 = torch.rand(4096, 4, device=dev); b2[:, 2:] += b2[:, :2]
    for name, fn in (("diou_loss", B.diou_loss), ("ciou_loss", B.ciou_loss), ("box_giou", B.box_giou)):
        row(f"{name} fwd", [4096, 4096], _time(lambda: fn(b1, b2), flush), (4096 + 4096) * 16 + 4096 * 4096 * 4, l2="L2 flushed")
    # ---- optimizers on the RepVGG-A1 parameter set (31.4 M parameters, 208 tensors)
    torch.manual_seed(0)
    model = hb.models.repvgg_a1(num_classes=1000).to(dev)
    params = [p for p in model.parameters()]
    for p in params:
        p.grad = torch.randn_like(p) * 1e-2
    np_ = sum(p.numel() for p in params)
    # algorithmic bytes / parameter: state tensors read + written once per pass (two passes where a per-tensor norm gates the
    # update: LAMB, TAdam, AdamP, RaLars 40 = 24 + 16; LARS without momentum 8 + 12)
    for name, cls, per in (("AdaBelief.step", hb.optim.AdaBelief, 28), ("LAMB.step", hb.optim.LAMB, 40), ("TAdam.step", hb.optim.TAdam, 40),
                           ("AdamP.step", hb.optim.AdamP, 40), ("Adan.step", hb.optim.Adan, 40), ("AdEMAMix.step", hb.optim.AdEMAMix, 36),
                           ("LARS.step", hb.optim.LARS, 20), ("RaLars.step", hb.optim.RaLars, 40)):
        opt = cls(params, lr=1e-4)
        row(name, [len(params), np_], _time(opt.step, flush), per * np_, l2="L2 flushed")
        del opt
    la = hb.optim.wrapper.Lookahead(torch.optim.SGD(params, lr=1e-4))
    row("Lookahead.sync_params", [len(params), np_], _time(lambda: la.sync_params(0.5), flush), 16 * np_, l2="L2 flushed")
    del la
    del model, params
    # ---- NormConv2d / Add2d (CUDA-core kernels: report FLOP-equivalents as well) and DropBlock
    x = torch.randn(32, 64, 56, 56, device=dev)
    w = torch.randn(64, 64, 3, 3, device=dev) * 0.05
    fl = 2.0 * 32 * 56 * 56 * 64 * 64 * 9
    byts = (x.numel() + 32 * 64 * 56 * 56 + w.numel()) * 4
    row("norm_conv2d fwd", [32, 64, 56, 56, 64, 3], _time(lambda: F.norm_conv2d(x, w, None, 1, 1), flush), byts, fl, "L2 flushed")
    row("add2d fwd", [32, 64, 56, 56, 64, 3], _time(lambda: F.add2d(x, w, None, 1, 1), flush), byts, fl, "L2 flushed")
    del x, w
    x = torch.randn(64, 256, 64, 64, device=dev, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    row("dropblock2d fwd", list(x.shape), _time(lambda: F.dropblock2d(x, 0.1 / 49, 7, False, True)), 2 * 2 * x.numel())
    return {"metric": "leaf-kernel micro rows (achieved GB/s over algorithmic bytes vs measured HBM peak)", "unit": "GB/s",
            "peak_hbm_gbs": peaks["hbm_gbs"], "peak_source": peaks["src"], "rows": rows,
            "timing": "CUDA events around the public API call with the stream parked behind a spin kernel (GPU time only), "
                      "3 warm-up + 10 timed iterations"}
