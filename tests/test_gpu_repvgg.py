"""GPU parity tests for the RepVGG path (BASELINE.json configs 0 and the N=1 bench workload): golden fixtures of the
reference's RepBlock forward/backward, config-1 argmax parity, training-step loss parity with the CPU oracle."""
import pytest
import torch
import torch.nn.functional as TF

import holocron_b200 as hb
from holocron_b200.models.classification.repvgg import RepBlock
from oracle.models import RepVGGOracle

from conftest import load_golden

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


@pytest.mark.parametrize("tag,cfg", [("s1", (16, 16, 1, True)), ("s2", (16, 32, 2, False))])
def test_repblock_vs_reference_golden(tag, cfg):
    d = load_golden("models")[f"repblock_{tag}"]
    blk = RepBlock(*cfg)
    blk.load_state_dict(d["state"])
    blk = blk.cuda().train()
    x = d["x"].cuda().requires_grad_(True)
    y = blk(x)
    (y.float() * d["up"].cuda()).sum().backward()
    assert rel_l2(y, d["y"]) < 6e-3                      # bf16 activations
    assert rel_l2(x.grad, d["gx"]) < 2e-2
    for n, p in blk.named_parameters():
        assert rel_l2(p.grad, d["grads"][n]) < 2e-2, n
    sd = blk.state_dict()
    for k in d["state_after"]:
        if "running" in k:
            assert rel_l2(sd[k], d["state_after"][k]) < 5e-3, k
        if "num_batches_tracked" in k:
            assert int(sd[k]) == int(d["state_after"][k])
    blk.eval()
    with torch.no_grad():
        assert rel_l2(blk(d["x"].cuda()), d["y_eval"]) < 6e-3
        blk.reparametrize()
        assert isinstance(blk.branches, torch.nn.Conv2d)
        assert rel_l2(blk.branches.weight, d["rep_w"]) < 1e-4 and rel_l2(blk.branches.bias, d["rep_b"]) < 1e-4
        assert rel_l2(blk(d["x"].cuda()), d["y_reparam"]) < 6e-3


def test_config1_argmax_parity():
    """BASELINE.json configs[0]: repvgg_a0, seed 0, x = rand(1,3,224,224): class argmax equal to the reference's
    (205), train-form eval and re-parametrised, logits within bf16 accuracy."""
    c = load_golden("models")["cfg1"]
    torch.manual_seed(0)
    m = hb.models.repvgg_a0(num_classes=1000).eval()
    x = torch.rand(1, 3, 224, 224)
    m = m.cuda()
    with torch.no_grad():
        lo = m(x.cuda())
        m.reparametrize()
        lr = m(x.cuda())
    assert not any(isinstance(mod, torch.nn.BatchNorm2d) for mod in m.modules())   # reference test_repvgg_reparametrize
    assert all(mod.kernel_size == (3, 3) for mod in m.modules() if isinstance(mod, torch.nn.Conv2d))
    assert int(lo.argmax()) == c["argmax"] and int(lr.argmax()) == c["argmax_rep"]
    assert rel_l2(lo, c["logits"]) < 3e-2 and rel_l2(lr, c["logits_rep"]) < 3e-2


def test_train_step_loss_parity_and_update():
    torch.manual_seed(0)
    m = hb.models.repvgg_a0(num_classes=1000)
    torch.manual_seed(0)
    o = RepVGGOracle("repvgg_a0", num_classes=1000)
    torch.manual_seed(1)
    x = torch.rand(4, 3, 224, 224)
    t = torch.randint(0, 1000, (4,))
    o.train()
    lo = TF.cross_entropy(o(x), t, label_smoothing=0.1)
    m = m.cuda().train()
    opt = hb.optim.AdaBelief(m.parameters(), lr=1e-3, betas=(0.95, 0.99), eps=1e-6)
    lm = TF.cross_entropy(m(x.cuda()), t.cuda(), label_smoothing=0.1)
    lm.backward()
    # bf16 forward through 28 blocks: loss within 1e-2 relative of the fp32 oracle
    assert abs(lm.item() - lo.item()) / abs(lo.item()) < 1e-2
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.parameters())
    before = [p.detach().clone() for p in m.parameters()]
    opt.step()
    assert all(not torch.equal(a, b) for a, b in zip(before, m.parameters()))
    # state_dict stays interchangeable with the oracle / reference layout
    o.load_state_dict({k: v.cpu() for k, v in m.state_dict().items()})


def test_cuda_graph_train_step_matches_eager():
    """holocron_b200.graphs.GraphedTrainStep: replaying the captured step (forward + CE + backward + AdaBelief with a
    device-side step counter) gives the same losses and parameters, bit for bit, as launching every kernel eagerly with
    the same history (2 warm-up steps on the first batch; the capture itself records without executing). Both arms use
    the capturable optimizer; no kernel of the step sums in an order that depends on scheduling. The optimizer states and
    BatchNorm buffers of three models are held to the same rule in test_gpu_grad_bucket_bounds.py."""
    from holocron_b200.distributed import GradBucket
    from holocron_b200.graphs import GraphedTrainStep

    torch.manual_seed(1)
    xs = [torch.rand(8, 3, 64, 64, device="cuda") for _ in range(3)]
    ts = [torch.randint(0, 10, (8,), device="cuda") for _ in range(3)]

    def build():
        torch.manual_seed(0)
        m = hb.models.repvgg_a0(num_classes=10).cuda().to(memory_format=torch.channels_last).train()
        bucket = GradBucket(m.parameters())
        opt = hb.optim.AdaBelief(m.parameters(), lr=1e-3, betas=(0.95, 0.99), eps=1e-6, capturable=True)

        def step(x, t):
            loss = TF.cross_entropy(m(x), t, label_smoothing=0.1)
            loss.backward()
            opt.step()
            bucket.zero_()
            return loss
        return m, step

    m_e, step_e = build()
    for _ in range(2):
        step_e(xs[0], ts[0])
    losses_e = [step_e(x, t).clone() for x, t in zip(xs, ts)]

    m_g, step_g = build()
    graphed = GraphedTrainStep(step_g, (xs[0], ts[0]), warmup=2)
    assert graphed.launches_per_replay > 100
    losses_g = [graphed(x, t).clone() for x, t in zip(xs, ts)]
    for a, b in zip(losses_g, losses_e):
        assert a.view(torch.int32).item() == b.view(torch.int32).item(), (losses_g, losses_e)
    for (n, a), b in zip(m_g.named_parameters(), m_e.parameters()):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), n
    assert losses_g[0].item() != losses_g[1].item()   # the replays really consumed the new inputs / updated parameters
