"""One fused step of every multi-tensor optimizer kernel (holocron_b200/csrc/optim.cu) from random NON-zero state,
checked per element against the fp64 steps and bounds of tests/_optim_oracle.py: every tensor the kernel writes (parameter,
state, the gradient for LARS with weight decay, the per-tensor scalars), and bit-equality of every tensor it must not
write. Sizes sit on each side of the chunk and vector edges, tables mix tiny and large tensors, and views at element offsets
1..3 take the kernels' scalar path, which tensors straight from the caching allocator never reach."""
import math

import pytest
import torch

import holocron_b200 as hb
import _optim_oracle as O
from holocron_b200._lib import lib
from holocron_b200.optim._multi_tensor import effective_strides

pytestmark = pytest.mark.gpu

CLASSES = {"adabelief": "AdaBelief", "lamb": "LAMB", "tadam": "TAdam", "adamp": "AdamP", "adan": "Adan",
           "ademamix": "AdEMAMix", "lars": "LARS", "ralars": "RaLars"}
SENTINEL = 12345.0
PAD = 4            # guard elements before a view (16 bytes, so that offset 0 stays on the vector path)
CASES = [(name, i) for name in O.STEPS for i in range(len(O.MODES[name]))]
# the mode of each optimizer with the most terms switched on, for the tests that are about tables and layouts
RICH = {"adabelief": 3, "adamp": 3, "tadam": 5, "adan": 3, "ademamix": 1, "lamb": 1, "ralars": 6,
        "lars": next(i for i, (k, _) in enumerate(O.MODES["lars"])
                     if k["weight_decay"] and k.get("dampening") and not k["first"])}


def _chunk():
    return lib().hb_optim_chunk_elems()


def _opt(name, params, kw, **extra):
    return getattr(hb.optim, CLASSES[name])(params, **{k: v for k, v in kw.items() if k != "first"}, **extra)


class Param:
    """The tensors of one parameter on the device (optionally as views at element offsets into sentinel-filled flat
    buffers), a bit copy of them from before the step, and the leaf handed to the optimizer."""

    def __init__(self, t, offsets=None, convert=None):
        self.bufs, self.dev = {}, {}
        for k, v in t.items():
            if offsets is None or v.numel() != t["p"].numel() or k == "W_t":
                d = v.cuda()
                self.dev[k] = convert(d) if convert is not None and v.shape == t["p"].shape and k != "W_t" else d
                continue
            buf = torch.full((v.numel() + 2 * PAD,), SENTINEL, device="cuda")
            o = PAD + offsets[k]
            self.bufs[k] = (buf, o, v.numel())
            self.dev[k] = buf[o:o + v.numel()].view(v.shape)
            self.dev[k].copy_(v)
        self.snapshot()
        self.p = self.dev["p"].requires_grad_()
        if "g" in self.dev:
            self.p.grad = self.dev["g"]

    def snapshot(self):
        self.before = {k: v.detach().clone() for k, v in self.dev.items()}

    def plant(self, opt, name, kw, step):
        st = {} if name == "lars" else {"step": step - 1}
        for k in O.state_keys(name, kw) + (("W_t",) if name == "tadam" else ()):
            st[k] = self.dev[k]
        if name in ("lamb", "ralars"):        # NaN: a trust ratio that is not written does not pass
            st["local_lr"] = self.dev["local_lr"] = torch.full((), math.nan, device="cuda")
        opt.state[self.p] = st

    def verify(self, opt, name, kw, step, what):
        """Checks every written tensor against the oracle's bound, every other one and the guards for bit-equality."""
        out, info = O.STEPS[name](self.before, step, kw, dev="cuda")
        got = dict(self.dev)
        got["p"] = self.p.detach()
        if name == "lars" and "momentum_buffer" in out and "momentum_buffer" not in got:
            got["momentum_buffer"] = opt.state[self.p]["momentum_buffer"]       # created by this step
        if self.p.numel():
            O.check(got, out, what)
            if name == "adamp":       # the projection was decided far from its threshold, or the case is badly built
                assert abs(info["margin"]) > 100 * info["margin_err"], f"{what}: margin {info['margin']:.3e}"
        for k, v in self.before.items():
            if k not in out:
                assert torch.equal(self.dev[k], v), f"{what}: {k} was written"
        for k, (buf, o, n) in self.bufs.items():
            assert bool((buf[:o] == SENTINEL).all()) and bool((buf[o + n:] == SENTINEL).all()), f"{what}: wrote outside {k}"
        return info


def _run(name, kw, step, tensors, what, offsets=None, convert=None, **extra):
    """One optimizer over one group holding ``tensors`` (CPU dicts), state planted, one step, every parameter verified."""
    ps = [Param(t, offsets, convert) for t in tensors]
    opt = _opt(name, [q.p for q in ps], kw, **extra)
    for q in ps:
        q.plant(opt, name, kw, step)
    opt.step()
    torch.cuda.synchronize()
    return [q.verify(opt, name, kw, step, f"{name} {what} [{i}] numel {q.p.numel()}") for i, q in enumerate(ps)], ps, opt


def _lookahead(kw, t, what, offsets=None):
    q = Param(t, offsets)
    la = hb.optim.wrapper.Lookahead(torch.optim.SGD([q.p], lr=0.1), sync_rate=kw["sync_rate"])
    la.param_groups[0]["params"][0] = q.dev["slow"]
    la.sync_params(kw["sync_rate"])
    torch.cuda.synchronize()
    q.verify(la, "lookahead", kw, 1, f"lookahead {what}")


def _side(name, i):
    return ("project", "keep")[i % 2] if name == "adamp" else None


def _expect(name, kw, step, infos, sizes):
    """The branches the case was built to take were taken."""
    big = [info for info, n in zip(infos, sizes) if n >= 255]
    if kw.get("amsgrad"):
        assert all(0.1 < info["max_kept"] < 0.9 for info in big)        # the maximum is kept here and replaced there
    if name in ("lamb", "ralars"):
        want = {O.CLIP_BELOW: -1, O.CLIP_ABOVE: 1, O.CLIP_NONE: 0}[kw["scale_clip"]]
        assert all(info["clip"] == want for info in big)
    if name == "ralars":
        assert {info["mode"] for info in infos} == {O.ralars_mode(step, kw["betas"][1], kw["force_adaptive_momentum"])[0]}
    if name == "adamp":
        assert {info["project"] for info in big} == {True, False}


# ---------------------------------------------------------------------------------------------------------------------
# a. sizes, every optimizer, every mode
@pytest.mark.parametrize("name,mode", CASES)
def test_single_tensor_sizes(name, mode):
    kw, step = O.MODES[name][mode]
    sizes, infos = O.sizes(_chunk()), []
    for i, n in enumerate(sizes):
        gen = torch.Generator().manual_seed(1000 * mode + i)
        t = O.random_tensors(name, (n,), kw, gen, side=_side(name, i))
        if name == "lookahead":
            _lookahead(kw, t, f"mode {mode} numel {n}")
        else:
            infos += _run(name, kw, step, [t], f"mode {mode}")[0]
    if name != "lookahead":
        _expect(name, kw, step, infos, sizes)


# ---------------------------------------------------------------------------------------------------------------------
# b. one table, many tensors (and g. the same launch twice)
def _table(name, kw):
    gen = torch.Generator().manual_seed(11)
    return [O.random_tensors(name, (n,), kw, gen, scale=O.table_scale(i), side=_side(name, i))
            for i, n in enumerate(O.table_sizes(_chunk()))]


@pytest.mark.parametrize("name", O.OPTIMIZERS)
def test_many_tensor_table(name):
    """chunks[blockIdx.x] -> (tensor, chunk) and the 2t / 4t / t scratch slots: per-tensor scales from 1e-3 to 1e2 make a
    reduction that lands in a neighbour's slot change the neighbour's trust ratio by orders of magnitude."""
    kw, step = O.MODES[name][RICH[name]]
    tensors = _table(name, kw)
    infos, ps, opt = _run(name, kw, step, tensors, "table")
    _expect(name, kw, step, infos, [t["p"].numel() for t in tensors])
    if name == "adamp":
        table, = opt._tables.values()
        assert table.num_tensors == len(tensors) and table.scratch.numel() >= 4 * len(tensors)


@pytest.mark.parametrize("name", ["lamb", "adamp"])
def test_reductions_repeat_bit_for_bit(name):
    """The per-tensor sums add fp64 partials atomically, in no fixed order; rounded to fp32 they are expected to come out
    the same from run to run. Two launches over the many-tensor table from identical state."""
    kw, step = O.MODES[name][RICH[name]]
    tensors = _table(name, kw)
    runs = [_run(name, kw, step, tensors, "repeat")[1] for _ in range(2)]
    for i, (a, b) in enumerate(zip(*runs)):
        for k in a.dev if a.p.numel() else ():          # a zero-element tensor has no chunk: nothing writes its scalar
            diff = (a.dev[k].double() - b.dev[k].double()).abs().max().item() if a.dev[k].numel() else 0.0
            assert torch.equal(a.dev[k], b.dev[k]), f"{name} tensor {i} {k}: runs differ by {diff:.3e}"


# ---------------------------------------------------------------------------------------------------------------------
# c. alignment
@pytest.mark.parametrize("name,mode", CASES)
def test_misaligned_views_take_the_scalar_path_within_the_same_bound(name, mode):
    kw, step = O.MODES[name][mode]
    for n in O.alignment_sizes(_chunk()):
        for ci, offsets in enumerate(O.alignment_cases(name, kw)):
            gen = torch.Generator().manual_seed(n + ci)
            t = O.random_tensors(name, (n,), kw, gen, side=_side(name, ci))
            if name == "lookahead":
                _lookahead(kw, t, f"offsets {offsets}", offsets)
                continue
            _, (q,), _ = _run(name, kw, step, [t], f"mode {mode} offsets {offsets}", offsets)
            for k, o in offsets.items():
                if k in q.dev:
                    assert q.dev[k].data_ptr() % 16 == 4 * o


# ---------------------------------------------------------------------------------------------------------------------
# d. zero norms and empty work
@pytest.mark.parametrize("zero", ["p", "g", "both"])
@pytest.mark.parametrize("name", ["lamb", "lars", "ralars", "adamp"])
def test_zero_norms(name, zero):
    kw, step = O.MODES[name][0]
    kw = {k: v for k, v in kw.items() if k != "scale_clip"}          # the default clip (0, 10) lets a zero norm through
    n = 2 * _chunk() + 3
    t = O.random_tensors(name, (n,), kw, torch.Generator().manual_seed(5))
    for k in t:
        if (k == "p" and zero != "g") or (k != "p" and zero != "p"):     # "g": zero gradient AND zero state
            t[k] = torch.zeros_like(t[k])
    (info,), (q,), opt = _run(name, kw, step, [t], f"zero {zero}")
    assert all(bool(torch.isfinite(v).all()) for v in q.dev.values())
    if name == "adamp":
        assert info["project"]         # the cosine of a zero vector is 0: k = (1 / eps)^2 * 0 must stay 0
    else:
        local_lr = q.dev["local_lr"] if name != "lars" else info["local_lr"].v
        assert float(local_lr) == 1.0


@pytest.mark.parametrize("name", O.OPTIMIZERS)
def test_parameters_without_gradient_are_left_out(name):
    kw, step = O.MODES[name][RICH[name]]
    C = _chunk()
    tensors = [O.random_tensors(name, (n,), kw, torch.Generator().manual_seed(n)) for n in (C + 1, 7, 2 * C)]

    def build(which, with_grad):
        ps = [Param(tensors[i]) for i in which]
        opt = _opt(name, [q.p for q in ps], kw)
        for i, q in zip(which, ps):
            q.plant(opt, name, kw, step)
            if i not in with_grad:
                q.p.grad = None
        opt.step()
        torch.cuda.synchronize()
        return ps

    for q in build((0, 1, 2), ()):                        # nothing to do: nothing is touched
        assert all(torch.equal(v, q.before[k]) for k, v in q.dev.items() if k != "local_lr")
    full, only = build((0, 1, 2), (0, 2)), build((0, 2), (0, 2))
    assert all(torch.equal(v, full[1].before[k]) for k, v in full[1].dev.items() if k != "local_lr")
    for a, b in zip((full[0], full[2]), only):
        assert all(torch.equal(a.dev[k], b.dev[k]) for k in a.dev)
        assert not torch.equal(a.dev["p"], a.before["p"])


# ---------------------------------------------------------------------------------------------------------------------
# e. host dispatch
@pytest.mark.parametrize("name", O.OPTIMIZERS)
def test_two_groups_each_with_its_own_hyper_parameters(name):
    kw_a, step = O.MODES[name][RICH[name]]
    kw_b = {**kw_a, "lr": 3 * kw_a["lr"], "weight_decay": 0.0 if name != "lars" else 5e-2}
    if "betas" in kw_b:
        kw_b["betas"] = tuple(0.5 + b / 2 for b in kw_a["betas"]) if name != "ralars" else (0.75, 255 / 256)
    if name == "lars":
        kw_b["momentum"] = 0.5
    n = _chunk() + 5
    qa, qb = (Param(O.random_tensors(name, (n,), kw, torch.Generator().manual_seed(s))) for s, kw in ((1, kw_a), (2, kw_b)))
    opt = _opt(name, [{"params": [qa.p]}, {"params": [qb.p], **{k: kw_b[k] for k in kw_b if kw_b[k] != kw_a[k]}}], kw_a)
    qa.plant(opt, name, kw_a, step)
    qb.plant(opt, name, kw_b, step)
    opt.step()
    torch.cuda.synchronize()
    qa.verify(opt, name, kw_a, step, f"{name} group 0")
    qb.verify(opt, name, kw_b, step, f"{name} group 1")


@pytest.mark.parametrize("name,capturable", [(n, False) for n in ("adabelief", "tadam", "adamp", "adan", "ademamix", "ralars")]
                         + [(n, True) for n in ("adabelief", "adamp", "adan")])
def test_one_group_at_different_step_counts(name, capturable):
    """Each parameter gets the bias corrections of its own count, and the tables (and device counters) are keyed by
    something that does not change from call to call."""
    kw, _ = O.MODES[name][RICH[name]]
    steps = (3, 7, 3)
    ps = [Param(O.random_tensors(name, (n,), kw, torch.Generator().manual_seed(n))) for n in (_chunk() + 1, 300, 5)]
    opt = _opt(name, [q.p for q in ps], kw, **({"capturable": True} if capturable else {}))
    for q, s in zip(ps, steps):
        q.plant(opt, name, kw, s)
    opt.step()
    torch.cuda.synchronize()
    infos = [q.verify(opt, name, kw, s, f"{name} at step {s}") for q, s in zip(ps, steps)]
    if name == "ralars":
        assert infos[0]["mode"] != infos[1]["mode"]
    for _ in range(20):
        opt.step()
    assert len(opt._tables) <= len(set(steps))
    assert [opt.state[q.p]["step"] for q in ps] == [s + 20 for s in steps]
    if capturable:
        assert len(opt._step_dev) <= len(set(steps))
        assert sorted(int(c) for c in opt._step_dev.values()) == sorted(s + 20 for s in set(steps))


def _channels_last(v):
    return v.contiguous(memory_format=torch.channels_last)


def _permuted(v):
    return v.t().contiguous().t()


@pytest.mark.parametrize("layout", ["channels_last", "permuted"])
@pytest.mark.parametrize("name", O.OPTIMIZERS)
def test_dense_layouts_other_than_contiguous(name, layout):
    kw, step = O.MODES[name][RICH[name]]
    shape, convert = ((16, 24, 5, 5), _channels_last) if layout == "channels_last" else ((130, 70), _permuted)
    t = O.random_tensors(name, shape, kw, torch.Generator().manual_seed(9))
    _, (q,), _ = _run(name, kw, step, [t], layout, convert=convert)
    assert not q.p.is_contiguous() and q.p.numel() == math.prod(shape)


@pytest.mark.parametrize("name", O.OPTIMIZERS)
def test_inputs_the_tensor_table_refuses(name):
    kw, _ = O.MODES[name][0]
    strided = torch.randn(64, device="cuda")[::2].requires_grad_()
    strided.grad = torch.randn(32, device="cuda")
    with pytest.raises(RuntimeError, match="share one dense memory layout"):
        _opt(name, [strided], kw).step()
    half = torch.randn(32, device="cuda", dtype=torch.float16).requires_grad_()
    half.grad = torch.randn(32, device="cuda", dtype=torch.float16)
    with pytest.raises(TypeError, match="float32"):
        _opt(name, [half], kw).step()


@pytest.mark.parametrize("name", O.OPTIMIZERS)
def test_gradient_in_another_layout(name):
    """Same result as the same gradient converted beforehand; LARS with weight decay leaves g + wd p in p.grad, in the
    parameter's layout."""
    kw, step = O.MODES[name][RICH[name]]
    t = O.random_tensors(name, (16, 24, 5, 5), kw, torch.Generator().manual_seed(13))
    (_,), (want,), _ = _run(name, kw, step, [t], "channels_last gradient")
    q = Param(t)
    q.p.grad = _channels_last(q.dev["g"])
    opt = _opt(name, [q.p], kw)
    q.plant(opt, name, kw, step)
    opt.step()
    torch.cuda.synchronize()
    for k in want.dev:
        if k != "g":
            assert torch.equal(q.dev[k], want.dev[k]), k
    if name == "lars":
        assert q.p.grad.dtype == torch.float32 and effective_strides(q.p.grad) == effective_strides(q.p)
        assert torch.equal(q.p.grad, want.p.grad) and not torch.equal(q.p.grad, want.before["g"])


# ---------------------------------------------------------------------------------------------------------------------
# f. device step counter and control block
def _regrad(q, seed):
    q.dev["g"].copy_(torch.randn(q.dev["g"].shape, generator=torch.Generator().manual_seed(seed)).cuda() * 0.1)
    q.snapshot()


@pytest.mark.parametrize("name", ["adabelief", "adamp", "adan"])
def test_device_step_counter_follows_three_steps(name):
    kw, step = O.MODES[name][RICH[name]]
    q = Param(O.random_tensors(name, (2 * _chunk() + 3,), kw, torch.Generator().manual_seed(3), side="project"))
    opt = _opt(name, [q.p], kw, capturable=True)
    q.plant(opt, name, kw, step)
    for s in range(step, step + 3):
        opt.step()
        torch.cuda.synchronize()
        q.verify(opt, name, kw, s, f"{name} capturable step {s}")
        assert [int(c) for c in opt._step_dev.values()] == [s]
        _regrad(q, s)


def _control_block(lr, beta1=-1.0, skip=0):
    """The device control block as holocron_b200/trainer/core.py builds it and ``apply_ctl`` of optim.cu reads it: fp32
    word 0 the learning rate, word 1 beta1 (negative: keep the group's), word 2, read as an integer, the skip flag."""
    ctl = torch.zeros(lib().hb_train_ctl_bytes() // 4, device="cuda", dtype=torch.float32)
    ctl[0], ctl[1] = lr, beta1
    ctl.view(torch.int32)[2] = skip
    return ctl


@pytest.mark.parametrize("name", ["adabelief", "adamp", "adan", "ademamix"])
def test_control_block(name):
    kw, step = O.MODES[name][RICH[name]]
    capturable = name != "ademamix"          # AdEMAMix reads the block but keeps its step count on the host
    extra = {"capturable": True} if capturable else {}
    t = O.random_tensors(name, (2 * _chunk() + 3,), kw, torch.Generator().manual_seed(4), side="project")
    # the block's learning rate replaces the group's; beta1 only when word 1 is not negative
    for beta1 in ((-1.0, 0.5) if capturable else (-1.0,)):
        q = Param(t)
        opt = _opt(name, [q.p], kw, **extra)
        q.plant(opt, name, kw, step)
        opt._hb_ctl = _control_block(2.5e-3, beta1)
        opt.step()
        torch.cuda.synchronize()
        used = {**kw, "lr": 2.5e-3}
        if beta1 >= 0:
            used["betas"] = (beta1,) + tuple(kw["betas"][1:])
        q.verify(opt, name, used, step, f"{name} control block beta1 {beta1}")
    # skip: nothing moves, the device counter included; clearing the flag resumes from the unadvanced count
    q = Param(t)
    opt = _opt(name, [q.p], kw, **extra)
    q.plant(opt, name, kw, step)
    opt._hb_ctl = _control_block(2.5e-3, skip=1)
    opt.step()
    torch.cuda.synchronize()
    assert all(torch.equal(v, q.before[k]) for k, v in q.dev.items())
    if capturable:
        assert [int(c) for c in opt._step_dev.values()] == [step - 1]
    opt._hb_ctl.view(torch.int32)[2] = 0
    opt.step()
    torch.cuda.synchronize()
    q.verify(opt, name, {**kw, "lr": 2.5e-3}, step if capturable else step + 1, f"{name} after a skipped step")
    if capturable:
        assert [int(c) for c in opt._step_dev.values()] == [step]


@pytest.mark.parametrize("name", O.OPTIMIZERS)
def test_optimizers_off_the_device_path_are_those_that_ignore_the_block(name):
    """LAMB, TAdam, LARS and RaLars never read the control block (a set skip flag does not stop them), and they are the
    ones the trainers keep off the device path, whatever a parameter group claims."""
    from holocron_b200.trainer.trainers import _reads_control_block
    kw, step = O.MODES[name][0]
    reads = name in ("adabelief", "adamp", "adan", "ademamix")
    q = Param(O.random_tensors(name, (300,), kw, torch.Generator().manual_seed(6)))
    opt = _opt(name, [q.p], kw)
    q.plant(opt, name, kw, step)
    for group in opt.param_groups:
        group["capturable"] = True
    assert _reads_control_block(opt) == reads
    opt._hb_ctl = _control_block(kw["lr"], skip=1)
    for group in opt.param_groups:
        group["capturable"] = False
    opt.step()
    torch.cuda.synchronize()
    assert torch.equal(q.dev["p"], q.before["p"]) == reads


# ---------------------------------------------------------------------------------------------------------------------
def test_functional_forms_meet_the_same_bound():
    C = _chunk()
    for name in ("adabelief", "tadam", "adamp", "adan", "ademamix"):
        kw, step = O.MODES[name][RICH[name]]
        ps = [Param(O.random_tensors(name, (n,), kw, torch.Generator().manual_seed(n), side="keep")) for n in (C + 5, 3)]
        col = lambda k: [q.dev[k] for q in ps] if k in ps[0].dev else []      # noqa: E731
        params, grads, steps = [q.p for q in ps], col("g"), [step] * len(ps)
        b, lr, wd, eps, ams = kw["betas"], kw["lr"], kw.get("weight_decay", 0.0), kw["eps"], kw.get("amsgrad", False)
        if name == "adabelief":
            hb.optim.adabelief(params, grads, col("exp_avg"), col("exp_avg_sq"), col("max_exp_avg_sq"), steps, ams, *b, lr, wd, eps)
        elif name == "tadam":
            hb.optim.tadam(params, grads, col("exp_avg"), col("exp_avg_sq"), col("max_exp_avg_sq"), col("W_t"), steps, ams, *b,
                           lr, wd, eps, kw.get("dof"))
        elif name == "adamp":
            hb.optim.adamp(params, grads, col("exp_avg"), col("exp_avg_sq"), col("max_exp_avg_sq"), steps, ams, *b, lr, wd, eps, 0.1)
        elif name == "adan":
            hb.optim.adan(params, grads, col("prev_grad"), col("exp_avg"), col("exp_avg_sq"), col("exp_avg_delta"),
                          col("max_exp_avg_delta"), steps, ams, *b, lr, wd, eps)
        else:
            hb.optim.ademamix(params, grads, col("exp_avg"), col("exp_avg_slow"), col("exp_avg_sq"), steps, *b, kw["alpha"], lr,
                              wd, eps)
        torch.cuda.synchronize()
        for q in ps:
            q.verify(None, name, kw, step, f"{name} functional")
    # a gradient of another dtype (autograd never assigns one to p.grad, the functional forms take what they are given)
    kw, step = O.MODES["adabelief"][0]
    t = O.random_tensors("adabelief", (C + 5,), kw, torch.Generator().manual_seed(8))
    t["g"] = t["g"].bfloat16().float()
    a, b = Param(t), Param(t)
    for q, g in ((a, a.dev["g"]), (b, b.dev["g"].bfloat16())):
        hb.optim.adabelief([q.p], [g], [q.dev["exp_avg"]], [q.dev["exp_avg_sq"]], [], [step], False, *kw["betas"], kw["lr"],
                           0.0, kw["eps"])
    torch.cuda.synchronize()
    a.verify(None, "adabelief", kw, step, "adabelief functional")
    assert all(torch.equal(a.dev[k], b.dev[k]) for k in a.dev)
