"""GPU parity tests for the fused optimizer steps (AdaBelief / LAMB / TAdam) against the reference's trajectories
(golden fixtures) and the CPU oracle. fp32 state: rtol 1e-4 (north_star allows 1e-3)."""
import pytest
import torch

import holocron_b200 as hb
import _optim_oracle as OB
from oracle import optim as OO

from conftest import load_golden

pytestmark = pytest.mark.gpu


def close(a, b, rtol=1e-4, atol=1e-6):
    torch.testing.assert_close(a.detach().cpu().float(), b.detach().cpu().float(), rtol=rtol, atol=atol)


@pytest.mark.parametrize("name,cls", [("adabelief", "AdaBelief"), ("adabelief_wd_ams", "AdaBelief"), ("lamb", "LAMB"),
                                      ("lamb_wd", "LAMB"), ("tadam", "TAdam"), ("tadam_wd_ams_dof", "TAdam")])
def test_trajectories_vs_reference(name, cls):
    g = load_golden("optim")
    params = [torch.nn.Parameter(p.clone().cuda()) for p in g["p0"]]
    opt = getattr(hb.optim, cls)(params, **g[name + "_kw"])
    for step in range(3):
        for p, gr in zip(params, g["grads"][step]):
            p.grad = gr.clone().cuda()
        opt.step()
        for p, ref in zip(params, g[name][step]):
            close(p, ref)
    st = opt.state[params[0]]
    assert st["step"] == 3 and isinstance(st["step"], int)
    assert set(st) >= {"step", "exp_avg", "exp_avg_sq"}
    if cls == "TAdam":
        assert st["W_t"].shape == (1,)
    if cls == "LAMB":
        assert "local_lr" in st
    # state_dict round trip keeps working (Optimizer protocol)
    sd = opt.state_dict()
    opt2 = getattr(hb.optim, cls)(params, **g[name + "_kw"])
    opt2.load_state_dict(sd)
    for p, gr in zip(params, g["grads"][0]):
        p.grad = gr.clone().cuda()
    opt2.step()


def test_adabelief_capturable_matches_default():
    """capturable=True (device-side step counter for CUDA-graph replay) follows the same trajectory."""
    g = load_golden("optim")
    params = [torch.nn.Parameter(p.clone().cuda()) for p in g["p0"]]
    opt = hb.optim.AdaBelief(params, capturable=True, **g["adabelief_kw"])
    for step in range(3):
        for p, gr in zip(params, g["grads"][step]):
            p.grad = gr.clone().cuda()
        opt.step()
        for p, ref in zip(params, g["adabelief"][step]):
            close(p, ref)


def test_optimizer_changes_params_like_reference_test():
    # reference tests/test_optim.py:10-39: one step on a 1024 -> 10 classifier layer must change its weight
    # (for TAdam the first update is ~1e-10 - the first w_t is (dof+d)/(sum(g^2)/eps) - so only tiny weights move,
    # exactly as in the reference)
    for cls, kw in ((hb.optim.AdaBelief, {}), (hb.optim.LAMB, {"weight_decay": 2e-5}), (hb.optim.TAdam, {})):
        torch.manual_seed(0)
        lin = torch.nn.Linear(1024, 10).cuda()
        opt = cls(lin.parameters(), lr=1e-4, **kw)
        before = lin.weight.data.clone()
        opt.zero_grad()
        loss = torch.nn.functional.cross_entropy(lin(torch.rand(4, 1024, device="cuda")), torch.zeros(4, dtype=torch.long, device="cuda"))
        loss.backward()
        opt.step()
        assert lin.weight.grad is not None
        assert not torch.equal(lin.weight.data, before), cls.__name__
        with pytest.raises(ValueError):
            cls(lin.parameters(), lr=-1.0)
        with pytest.raises(ValueError):
            cls(lin.parameters(), betas=(1.1, 0.9))


def test_functional_apis():
    torch.manual_seed(0)
    ps = [torch.randn(100, device="cuda"), torch.randn(7, 9, device="cuda")]
    gs = [torch.randn_like(p) for p in ps]
    ref_p = [p.cpu().clone() for p in ps]
    m = [torch.zeros_like(p) for p in ps]; v = [torch.zeros_like(p) for p in ps]
    hb.optim.adabelief(ps, gs, m, v, [], [1, 1], False, 0.9, 0.999, 1e-2, 0.0, 1e-8)
    for rp, g_ in zip(ref_p, gs):
        OO.adabelief_step(rp, g_.cpu(), torch.zeros_like(rp), torch.zeros_like(rp), 1, 1e-2, 0.9, 0.999, 1e-8)
    for a, b in zip(ps, ref_p):
        close(a, b)
    W = [0.9 / 0.1 * torch.ones(1, device="cuda") for _ in ps]
    ref2 = [p.cpu().clone() for p in ps]
    m = [torch.zeros_like(p) for p in ps]; v = [torch.zeros_like(p) for p in ps]
    hb.optim.tadam(ps, gs, m, v, [], W, [1, 1], False, 0.9, 0.999, 1e-2, 0.0, 1e-8, None)
    for rp, g_ in zip(ref2, gs):
        OO.tadam_step(rp, g_.cpu(), torch.zeros_like(rp), torch.zeros_like(rp), 0.9 / 0.1 * torch.ones(1), 1, 1e-2, 0.9, 0.999, 1e-8)
    for a, b in zip(ps, ref2):
        close(a, b)


def test_full_size_repvgg_a1_parameter_set_vs_oracle():
    """BASELINE config 3 optimizer: AdaBelief(lr=1e-3, betas=(0.95, 0.99), eps=1e-6) over RepVGG-A1's 208 tensors /
    31.4 M parameters; the CUDA step is compared with the oracle on every tensor (2 steps as whole tensors, the third per
    element from the oracle's state), plus channels_last
    parameter layouts and the step/linearity property p(lr=2a) - p0 == 2 (p(lr=a) - p0)."""
    torch.manual_seed(0)
    model = hb.models.repvgg_a1(num_classes=1000)
    shapes = [tuple(p.shape) for p in model.parameters()]
    assert len(shapes) == 208 and sum(torch.Size(s).numel() for s in shapes) > 31_000_000
    params = []
    for s in shapes:
        t = torch.randn(*s) * 0.05
        if len(s) == 4:
            t = t.contiguous(memory_format=torch.channels_last)
        params.append(t)
    dev = [torch.nn.Parameter(p.clone().cuda()) for p in params]
    kw = {"lr": 1e-3, "betas": (0.95, 0.99), "eps": 1e-6, "weight_decay": 1e-2}
    opt = hb.optim.AdaBelief(dev, **kw)
    cpu_m = [torch.zeros_like(p) for p in params]; cpu_s = [torch.zeros_like(p) for p in params]
    for step in range(1, 4):
        grads = [torch.randn_like(p) * 0.01 for p in params]
        if step == 3:
            # two steps in, the trajectories agree as whole tensors; the last step then starts from the oracle's state and
            # is held to the per-element bound of tests/_optim_oracle.py, parameter and both moments
            worst = max(((d.detach().cpu() - p).abs().max() / (p.abs().max() + 1e-12)).item() for d, p in zip(dev, params))
            assert worst < 1e-5, worst
            for d, p, m, s in zip(dev, params, cpu_m, cpu_s):
                d.data.copy_(p); opt.state[d]["exp_avg"].copy_(m); opt.state[d]["exp_avg_sq"].copy_(s)
            before = [{"p": d.detach().clone(), "g": g_.cuda(), "exp_avg": opt.state[d]["exp_avg"].clone(),
                       "exp_avg_sq": opt.state[d]["exp_avg_sq"].clone()} for d, g_ in zip(dev, grads)]
        for d, g_ in zip(dev, grads):
            d.grad = g_.cuda()
        opt.step()
        if step < 3:
            for p, g_, m, s in zip(params, grads, cpu_m, cpu_s):
                OO.adabelief_step(p, g_, m, s, step, kw["lr"], *kw["betas"], kw["eps"], kw["weight_decay"])
    for i, (d, t) in enumerate(zip(dev, before)):
        out, _ = OB.adabelief(t, 3, kw, dev="cuda")
        OB.check({"p": d.detach(), **{k: opt.state[d][k] for k in ("exp_avg", "exp_avg_sq")}}, out, f"tensor {i} {shapes[i]}")
    # linearity in lr of a single step from identical state
    p0 = torch.randn(100_003, device="cuda")
    g0 = torch.randn_like(p0)
    outs = []
    for lr in (1e-3, 2e-3):
        p = torch.nn.Parameter(p0.clone()); p.grad = g0.clone()
        hb.optim.AdaBelief([p], lr=lr).step()
        outs.append(p.detach() - p0)
    close(outs[1], 2 * outs[0], 1e-3, 1e-6)   # differences of fp32 parameters: quantised at ulp(p) ~ 1e-7


# ---------------------------------------------------------------------------------------------------------------------
# SURVEY §8 f2: Adan, AdEMAMix, LARS, RaLars, Lookahead - trajectories of the unmodified reference (tests/golden/optim2.pt)
OPTIM2 = [("adan", "Adan"), ("adan_wd_ams", "Adan"), ("ademamix", "AdEMAMix"), ("ademamix_wd", "AdEMAMix"), ("lars", "LARS"),
          ("lars_mom_wd", "LARS"), ("lars_nesterov", "LARS"), ("ralars", "RaLars"), ("ralars_rect_wd", "RaLars"),
          ("ralars_force", "RaLars")]


def _drive(opt, params, g, steps, keep):
    out = []
    for it in range(1, steps + 1):
        for p, p0, gr in zip(params, g["params"], g["grads"]):
            p.grad = (gr * it + 0.01 * p0).cuda()
        opt.step()
        if it in keep:
            out.append([p.detach().clone() for p in params])
    return out


@pytest.mark.parametrize("name,cls", OPTIM2)
def test_remaining_optimizers_vs_reference_trajectories(name, cls):
    g = load_golden("optim2")
    kw = g[name]["kw"]
    params = [torch.nn.Parameter(p.clone().cuda()) for p in g["params"]]
    opt = getattr(hb.optim, cls)(params, **kw)
    traj = _drive(opt, params, g, 6, (1, 3, 6))
    for ours, ref in zip(traj, g[name]["traj"]):
        for a, b in zip(ours, ref):
            close(a, b, 2e-4, 2e-6)
    st = opt.state[params[0]]
    if cls == "Adan":
        assert set(st) >= {"step", "exp_avg", "exp_avg_sq", "exp_avg_delta", "prev_grad"} and st["step"] == 6
        assert not st["prev_grad"].any()          # reference quirk: allocated, never written
        assert ("max_exp_avg_delta" in st) == bool(kw.get("amsgrad"))
    if cls == "AdEMAMix":
        assert set(st) == {"step", "exp_avg", "exp_avg_slow", "exp_avg_sq"}
    if cls == "LARS":
        assert ("momentum_buffer" in st) == (kw.get("momentum", 0.0) != 0)
        assert opt.scale_clip == (0.0, 10.0)
        if "grad_after" in g[name]:
            for p, want in zip(params, g[name]["grad_after"]):     # the weight decay lands IN the gradient, as in the reference
                close(p.grad, want, 1e-5, 1e-7)
    if cls == "RaLars":
        for p, want in zip(params, g[name]["local_lr"]):
            got = float(opt.state[p]["local_lr"])
            assert abs(got - want) <= 2e-4 * max(1.0, abs(want)), (got, want)
    # Optimizer protocol: state_dict round trip, then one more step
    opt2 = getattr(hb.optim, cls)(params, **kw)
    opt2.load_state_dict(opt.state_dict())
    for p in params:
        p.grad = torch.ones_like(p)
    opt2.step()


def test_remaining_optimizers_argument_validation_like_the_reference():
    w = [torch.nn.Parameter(torch.randn(4, 4, device="cuda"))]
    with pytest.raises(ValueError):
        hb.optim.LARS(w, lr=1)                      # the reference insists on a python float (lars.py:60)
    with pytest.raises(ValueError):
        hb.optim.LARS(w, lr=0.1, nesterov=True)     # needs momentum
    with pytest.raises(ValueError):
        hb.optim.AdEMAMix(w, betas=(0.9, 0.999, 1.0))
    with pytest.raises(ValueError):
        hb.optim.RaLars(w, eps=-1.0)
    with pytest.raises(ValueError):
        hb.optim.Adan(w, lr=-1.0)
    with pytest.raises(ValueError):
        hb.optim.wrapper.Lookahead(torch.optim.SGD(w, lr=0.1), sync_rate=1.5)
    with pytest.raises(ValueError):
        hb.optim.wrapper.Lookahead(torch.optim.SGD(w, lr=0.1), sync_period=0)
    assert isinstance(hb.optim.Adan(w), torch.optim.Adam)


def test_adan_functional_and_capturable():
    g = load_golden("optim2")
    kw = g["adan"]["kw"]
    params = [torch.nn.Parameter(p.clone().cuda()) for p in g["params"]]
    opt = hb.optim.Adan(params, capturable=True, **kw)
    traj = _drive(opt, params, g, 3, (1, 3))
    for ours, ref in zip(traj, g["adan"]["traj"][:2]):
        for a, b in zip(ours, ref):
            close(a, b, 2e-4, 2e-6)
    # functional form == one step of the oracle
    ps = [p.clone().cuda() for p in g["params"]]
    gs = [gr.clone().cuda() for gr in g["grads"]]
    z = lambda: [torch.zeros_like(p) for p in ps]       # noqa: E731
    hb.optim.adan(ps, gs, z(), z(), z(), z(), [], [1] * len(ps), False, 0.98, 0.92, 0.99, 1e-2, 0.0, 1e-8)
    for p, p0, gr in zip(ps, g["params"], g["grads"]):
        ref = p0.clone()
        OO.adan_step(ref, gr, torch.zeros_like(ref), torch.zeros_like(ref), torch.zeros_like(ref), torch.zeros_like(ref), 1, 1e-2,
                     0.98, 0.92, 0.99, 1e-8)
        close(p, ref, 2e-4, 2e-6)
    ps = [p.clone().cuda() for p in g["params"]]
    hb.optim.ademamix(ps, gs, z(), z(), z(), [2] * len(ps), 0.9, 0.99, 0.999, 5.0, 1e-2, 1e-2, 1e-8)
    for p, p0, gr in zip(ps, g["params"], g["grads"]):
        ref = p0.clone()
        OO.ademamix_step(ref, gr, torch.zeros_like(ref), torch.zeros_like(ref), torch.zeros_like(ref), 2, 1e-2, 0.9, 0.99, 0.999, 5.0,
                         1e-8, 1e-2)
        close(p, ref, 2e-4, 2e-6)


def test_lookahead_vs_reference_trajectory_and_state_dict():
    g = load_golden("optim2")
    params = [torch.nn.Parameter(p.clone().cuda()) for p in g["params"]]
    base = torch.optim.SGD(params, lr=0.1, momentum=0.9)
    la = hb.optim.wrapper.Lookahead(base, sync_rate=0.5, sync_period=3)
    traj = _drive(la, params, g, 7, (2, 3, 7))
    for ours, ref in zip(traj, g["lookahead"]["traj"]):
        for a, b in zip(ours, ref):
            close(a, b, 1e-5, 1e-6)
    for s, want in zip(la.param_groups[0]["params"], g["lookahead"]["slow"]):
        close(s, want, 1e-5, 1e-6)
    assert la.fast_steps == 7
    assert repr(la) == g["lookahead"]["repr"]
    sd = la.state_dict()
    assert "base_state_dict" in sd and "param_groups" in sd
    # sync_rate 0: the fast weights are reset to the slow ones
    for p in params:
        p.data.add_(1.0)
    la.sync_params(0.0)
    for p, s in zip(params, la.param_groups[0]["params"]):
        assert torch.equal(p.data, s)
    # the wrapper also drives the fused optimizers
    la2 = hb.optim.wrapper.Lookahead(hb.optim.AdaBelief(params, lr=1e-3), sync_period=2)
    for _ in range(4):
        for p in params:
            p.grad = torch.ones_like(p)
        la2.step()
    la2.zero_grad()
    assert all(p.grad is None for p in params)
