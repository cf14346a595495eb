"""Dev harness (GPU): RepBlock / RepVGG forward+backward through the CUDA path vs golden fixtures + oracle."""
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, ".")
import holocron_b200 as hb
from holocron_b200.models.classification.repvgg import RepBlock
from oracle.models import RepVGGOracle


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def check(name, a, b, tol):
    r = rel(a, b)
    print(f"{'OK ' if r < tol else 'BAD'} {name}: rel_l2={r:.3e} (tol {tol})", flush=True)
    return r < tol


def repblock_golden():
    g = torch.load("tests/golden/models.pt")
    ok = True
    for tag, (cin, cout, stride, ident) in (("s1", (16, 16, 1, True)), ("s2", (16, 32, 2, False))):
        d = g[f"repblock_{tag}"]
        blk = RepBlock(cin, cout, stride, ident)
        blk.load_state_dict(d["state"])
        blk = blk.cuda().train()
        x = d["x"].cuda().requires_grad_(True)
        y = blk(x)
        (y.float() * d["up"].cuda()).sum().backward()
        ok &= check(f"repblock {tag} y", y, d["y"], 1e-2)
        ok &= check(f"repblock {tag} gx", x.grad, d["gx"], 2e-2)
        for n, p in blk.named_parameters():
            ok &= check(f"repblock {tag} grad {n}", p.grad, d["grads"][n], 2e-2)
        sd = blk.state_dict()
        for k in ("branches.0.1.running_mean", "branches.0.1.running_var", "branches.1.1.running_var"):
            ok &= check(f"repblock {tag} {k}", sd[k], d["state_after"][k], 5e-3)
        blk.eval()
        with torch.no_grad():
            ye = blk(d["x"].cuda())
            ok &= check(f"repblock {tag} eval", ye, d["y_eval"], 1e-2)
            blk.reparametrize()
            yr = blk(d["x"].cuda())
            ok &= check(f"repblock {tag} reparam", yr, d["y_reparam"], 1e-2)
            ok &= check(f"repblock {tag} rep_w", blk.branches.weight, d["rep_w"], 1e-6)
    return ok


def config1():
    g = torch.load("tests/golden/models.pt")["cfg1"]
    torch.manual_seed(0)
    m = hb.models.repvgg_a0(num_classes=1000).eval()
    x = torch.rand(1, 3, 224, 224)
    m = m.cuda()
    with torch.no_grad():
        lo = m(x.cuda())
        m.reparametrize()
        lr = m(x.cuda())
    print("cfg1 argmax ours", int(lo.argmax()), int(lr.argmax()), "golden", g["argmax"], g["argmax_rep"])
    ok = int(lo.argmax()) == g["argmax"] and int(lr.argmax()) == g["argmax_rep"]
    ok &= check("cfg1 logits train-form", lo, g["logits"], 2e-2)
    ok &= check("cfg1 logits reparam", lr, g["logits_rep"], 2e-2)
    return ok


def train_parity(batch=8):
    torch.manual_seed(0)
    m = hb.models.repvgg_a0(num_classes=1000)
    torch.manual_seed(0)
    o = RepVGGOracle("repvgg_a0", num_classes=1000)
    torch.manual_seed(1)
    x = torch.rand(batch, 3, 224, 224)
    t = torch.randint(0, 1000, (batch,))
    o.train()
    lo = F.cross_entropy(o(x), t, label_smoothing=0.1)
    lo.backward()
    m = m.cuda().train()
    out = m(x.cuda())
    lm = F.cross_entropy(out, t.cuda(), label_smoothing=0.1)
    lm.backward()
    print(f"loss ours {lm.item():.6f} oracle {lo.item():.6f} rel {abs(lm.item()-lo.item())/abs(lo.item()):.3e}")
    ok = abs(lm.item() - lo.item()) / abs(lo.item()) < 5e-3
    po = dict(o.named_parameters())
    worst = 0
    for n, p in m.named_parameters():
        key = n
        r = rel(p.grad, po[key].grad)
        worst = max(worst, r)
    print("worst grad rel_l2 over all params:", worst)
    for n in ["head.weight", "features.4.1.branches.0.0.weight", "features.2.2.branches.0.0.weight", "features.0.0.branches.0.0.weight",
              "features.0.0.branches.0.1.weight", "features.3.5.branches.2.bias"]:
        print("  ", n, rel(dict(m.named_parameters())[n].grad, po[n].grad))
    return ok


def timing(batch=256, steps=10, name="repvgg_a0"):
    torch.manual_seed(0)
    m = getattr(hb.models, name)(num_classes=1000).cuda().train()
    opt = hb.optim.AdaBelief(m.parameters(), lr=1e-3, betas=(0.95, 0.99), eps=1e-6)
    x = torch.rand(batch, 3, 224, 224, device="cuda")
    t = torch.randint(0, 1000, (batch,), device="cuda")

    def step():
        out = m(x)
        loss = F.cross_entropy(out, t, label_smoothing=0.1)
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        return loss

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) / steps * 1e3
    ms = e0.elapsed_time(e1) / steps
    print(f"ours {name} b{batch}: {ms:.2f} ms/step (wall {wall:.2f}) -> {batch/ms*1e3:.0f} img/s, loss {loss.item():.4f}, "
          f"mem {torch.cuda.max_memory_allocated()/2**30:.1f} GiB")
    # forward only / fwd+bwd split
    for _ in range(2):
        with torch.no_grad():
            m(x)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        with torch.no_grad():
            m(x)
    e1.record()
    torch.cuda.synchronize()
    print(f"   fwd only (train-mode BN): {e0.elapsed_time(e1)/steps:.2f} ms")
    # torch eager reference on the same GPU (cuDNN, bf16 autocast, channels_last)
    torch.manual_seed(0)
    o = RepVGGOracle(name, num_classes=1000).cuda().train().to(memory_format=torch.channels_last)
    oopt = torch.optim.Adam(o.parameters(), lr=1e-3, fused=True)
    xc = x.contiguous(memory_format=torch.channels_last)

    def ostep():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = o(xc)
            loss = F.cross_entropy(out.float(), t, label_smoothing=0.1)
        loss.backward()
        oopt.step()
        oopt.zero_grad(set_to_none=True)

    for _ in range(3):
        ostep()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        ostep()
    e1.record()
    torch.cuda.synchronize()
    ms_o = e0.elapsed_time(e1) / steps
    print(f"torch eager (cuDNN bf16 autocast channels_last, fused Adam) {name} b{batch}: {ms_o:.2f} ms/step -> {batch/ms_o*1e3:.0f} img/s")


if __name__ == "__main__":
    print(torch.cuda.get_device_name(0))
    ok = repblock_golden()
    ok &= config1()
    ok &= train_parity(8)
    print("ALL OK" if ok else "SOME BAD")
    timing(256, 10)
    if "--profile" in sys.argv:
        from torch.profiler import profile, ProfilerActivity
        m = hb.models.repvgg_a0(num_classes=1000).cuda().train()
        opt = hb.optim.AdaBelief(m.parameters(), lr=1e-3)
        x = torch.rand(256, 3, 224, 224, device="cuda")
        t = torch.randint(0, 1000, (256,), device="cuda")
        for _ in range(2):
            F.cross_entropy(m(x), t).backward(); opt.step(); opt.zero_grad()
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            for _ in range(3):
                F.cross_entropy(m(x), t).backward(); opt.step(); opt.zero_grad()
            torch.cuda.synchronize()
        print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25))
