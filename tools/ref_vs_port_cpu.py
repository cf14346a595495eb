"""CPU check (needs a reference checkout, HOLOCRON_REFERENCE): the UNMODIFIED reference's RepVGG-A0 train step
(holocron.models.repvgg_a0 + holocron.optim.AdaBelief, CPU fp32) timed beside the oracle port that `bench.py --impl reference`
runs, which stands in for the reference arm where no reference checkout exists."""
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, ".")
from oracle import reference_loader
from oracle.models import RepVGGOracle
from oracle.optim import adabelief_step

holocron = reference_loader.load()
torch.set_num_threads(8)
g = torch.Generator().manual_seed(0)
x = torch.rand(8, 3, 224, 224, generator=g)
t = torch.randint(0, 1000, (8,), generator=g)


def time_steps(step, n=4):
    step(1)
    t0 = time.perf_counter()
    for i in range(n):
        step(2 + i)
    return (time.perf_counter() - t0) / n


torch.manual_seed(0)
ref = holocron.models.repvgg_a0(num_classes=1000).train()
opt = holocron.optim.AdaBelief(ref.parameters(), lr=1e-3, betas=(0.95, 0.99), eps=1e-6)
losses_ref = []


def ref_step(i):
    loss = F.cross_entropy(ref(x), t, label_smoothing=0.1)
    opt.zero_grad()
    loss.backward()
    opt.step()
    losses_ref.append(loss.item())


torch.manual_seed(0)
port = RepVGGOracle("repvgg_a0", num_classes=1000).train()
state = [(torch.zeros_like(p), torch.zeros_like(p)) for p in port.parameters()]
losses_port = []


def port_step(i):
    loss = F.cross_entropy(port(x), t, label_smoothing=0.1)
    loss.backward()
    for p, (m, s) in zip(port.parameters(), state):
        adabelief_step(p.data, p.grad, m, s, i, 1e-3, 0.95, 0.99, 1e-6)
        p.grad = None
    losses_port.append(loss.item())


tr, tp = time_steps(ref_step), time_steps(port_step)
print(f"reference (unmodified holocron): {tr * 1e3:.1f} ms / 8-image step = {8 / tr:.2f} images/s on {torch.get_num_threads()} threads")
print(f"oracle port                    : {tp * 1e3:.1f} ms / 8-image step = {8 / tp:.2f} images/s")
print("losses reference", [round(v, 5) for v in losses_ref])
print("losses port     ", [round(v, 5) for v in losses_port])
