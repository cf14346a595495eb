"""Teacher-forced parity hooks for whole-model GPU tests (test infrastructure).

A deep random-init network in training mode is ill-conditioned: batch-norm over a handful of samples re-normalises the
bf16 rounding noise at every layer, and end-to-end outputs of ANY bf16 execution drift from the fp32 fixture (torch's
own bf16 autocast lands 0.05 - 0.47 rel-L2 away on the Darknet fixtures). An
end-to-end tolerance alone therefore says little about kernel correctness. These hooks check, while the model runs,
EVERY fused launch against fp32 torch library ops applied to the very same input tensors (teacher forcing), so each
comparison spans exactly one unit and the tolerance can be tight (5e-3 rel-L2; the bf16 output rounding alone
is ~1.7e-3):

  * conv launches   - conv2d_forward_raw (all dense convolutions, incl. the data-gradient launches routed through it)
  * BN/act passes   - bn_act (statistics + normalise + residual + activation)
  * conv-BN-act     - conv_bn_act units from the fp32 MASTER weights (also covers filter packing / channel padding)
"""
import contextlib
import sys

import torch
import torch.nn.functional as TF

from holocron_b200.models import _blocks
from holocron_b200.nn import _fused


def _act_ref(z, act, slope):
    if act == 1:
        return z.relu()
    if act == 2:
        return z.clamp(0, 6)
    if act == 3:
        return TF.silu(z)
    if act == 4:
        return TF.leaky_relu(z, slope)
    if act == 5:
        return z * torch.tanh(TF.softplus(z))
    if act == 6:
        return 0.5 * z * (z + 2).clamp(0, 2)
    return z


def _rel(a, b):
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


def _bn_ref(u, bn, training):
    uf = u.detach().float()[:, :bn.num_features]
    if training or bn.running_mean is None:
        mean = uf.mean((0, 2, 3), keepdim=True)
        var = uf.var((0, 2, 3), unbiased=False, keepdim=True)
    else:
        mean, var = bn.running_mean.view(1, -1, 1, 1), bn.running_var.view(1, -1, 1, 1)
    w = 1.0 if bn.weight is None else bn.weight.detach().view(1, -1, 1, 1)
    b = 0.0 if bn.bias is None else bn.bias.detach().view(1, -1, 1, 1)
    return (uf - mean) / torch.sqrt(var + bn.eps) * w + b


class Report:
    def __init__(self):
        self.convs, self.bns, self.units = [], [], []

    def worst(self):
        return {k: max((e for _, e in getattr(self, k)), default=0.0) for k in ("convs", "bns", "units")}

    def assert_ok(self, conv_tol=5e-3, bn_tol=5e-3, unit_tol=5e-3):
        for name, tol in (("convs", conv_tol), ("bns", bn_tol), ("units", unit_tol)):
            bad = [(d, e) for d, e in getattr(self, name) if not e < tol]
            assert not bad, f"{name}: {len(bad)} launches off by more than {tol}: {bad[:5]}"


@contextlib.contextmanager
def teacher_forcing():
    rep = Report()
    orig_conv, orig_bn, orig_unit = _fused.conv2d_forward_raw, _fused.bn_act, _blocks.conv_bn_act

    def conv(x, wf, cout, r, s, stride, pad, dil, bias=None, residual=None, act=0, **kw):
        out = orig_conv(x, wf, cout, r, s, stride, pad, dil, bias=bias, residual=residual, act=act, **kw)
        y, y2 = out if isinstance(out, tuple) else (out, None)
        with torch.no_grad():
            ref = TF.conv2d(x.float(), wf[:cout].permute(0, 3, 1, 2).float(), None if bias is None else bias[:cout].float(),
                            stride, pad, dil)
            if kw.get("xe") is not None:      # K extension: a second 1x1 source in the same accumulator
                ref = ref + TF.conv2d(kw["xe"].float(), kw["we"][:cout].permute(0, 3, 1, 2).float())
            if residual is not None:
                ref = ref + residual.float()
            if act == 1:
                ref = ref.relu()
            rep.convs.append(((tuple(x.shape), tuple(wf.shape), stride, pad), _rel(y.float(), ref)))
            if y2 is not None:               # dual output: the 1x1 branch from the centre-tap loads
                ref2 = TF.conv2d(x.float(), kw["w2"][:cout].permute(0, 3, 1, 2).float(), None, stride, 0, dil)
                rep.convs.append(((tuple(x.shape), tuple(kw["w2"].shape), stride, 0), _rel(y2.float(), ref2)))
            if kw.get("want_stats"):         # epilogue statistics vs the stored bf16 output
                for t in (y, y2):
                    if t is None:
                        continue
                    parts, slots = _fused.get_stats(t)
                    tot = parts[:slots].double().sum(0)
                    tf = t.double()
                    ref_s = torch.stack([tf.sum((0, 2, 3)), (tf * tf).sum((0, 2, 3))], 1)
                    rep.convs.append((("stats", tuple(t.shape)), _rel(tot, ref_s)))
        return out

    def bn_act(us, bns, act=0, slope=0.0, residual=None, training=None, res_after_act=False, emit_stats=False):
        out = orig_bn(us, bns, act, slope, residual, training, res_after_act, emit_stats)
        with torch.no_grad():
            tr = bns[0].training if training is None else training
            z = sum(_bn_ref(u, bn, tr) for u, bn in zip(us, bns))
            c = bns[0].num_features
            if residual is not None and not res_after_act:
                r = residual.detach().float()[:, :c]
                z = torch.maximum(z, r) if act == 7 else z + r
            ref = _act_ref(z, act, slope)
            if residual is not None and res_after_act:
                ref = ref + residual.detach().float()[:, :c]
            rep.bns.append(((tuple(us[0].shape), len(us), act), _rel(out.detach().float()[:, :c], ref)))
        return out

    def unit(x, conv_m, bn, act, residual=None, res_after_act=False, keep_padded=False):
        out = orig_unit(x, conv_m, bn, act, residual, res_after_act, keep_padded)
        with torch.no_grad():
            wq = conv_m.weight.detach().to(torch.bfloat16).float()
            bq = None if conv_m.bias is None else conv_m.bias.detach().float()
            if type(conv_m).__name__ == "TridentConv2d":
                # one filter over three channel chunks, dilation 1 / 2 / 3 for the 3x3 layers (reference tridentnet.py:36-59)
                xf = x.detach().to(torch.bfloat16).float()
                dils = [1, 1, 1] if conv_m.dilation[0] == 1 else [1, 2, 3]
                z = torch.cat([TF.conv2d(c, wq, bq, conv_m.stride, tuple(d * p for p in conv_m.padding), (d, d), conv_m.groups)
                               for c, d in zip(torch.chunk(xf, 3, 1), dils)], 1)
            else:
                xf = x.detach()[:, :conv_m.in_channels].to(torch.bfloat16).float()   # the kernels' operand rounding
                z = TF.conv2d(xf, wq, bq, conv_m.stride, conv_m.padding, conv_m.dilation, conv_m.groups)
            if bn is not None:
                z = _bn_ref(z.to(torch.bfloat16), bn, bn.training)
            code, slope = _fused.act_code(act)
            c = z.shape[1]            # == conv_m.out_channels (3 x that behind a TridentConv2d)
            if residual is not None and not res_after_act:
                z = z + residual.detach().float()[:, :c]
            ref = _act_ref(z, code, slope)
            if residual is not None and res_after_act:
                ref = ref + residual.detach().float()[:, :c]
            rep.units.append(((tuple(x.shape), tuple(conv_m.weight.shape), conv_m.stride), _rel(out.detach().float()[:, :c], ref)))
        return out

    patched = []
    _fused.conv2d_forward_raw, _fused.bn_act = conv, bn_act
    for name, mod in list(sys.modules.items()):
        if name.startswith("holocron_b200.models") and getattr(mod, "conv_bn_act", None) is orig_unit:
            mod.conv_bn_act = unit
            patched.append(mod)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        yield rep
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
        _fused.conv2d_forward_raw, _fused.bn_act = orig_conv, orig_bn
        for mod in patched:
            mod.conv_bn_act = orig_unit
