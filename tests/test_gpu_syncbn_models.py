"""nn.SyncBatchNorm.convert_sync_batchnorm on the fused models.

* World size 1 or torch.distributed not initialised: a converted model runs the plain BatchNorm path, so its output,
  every gradient and the running statistics are bit-identical to the unconverted model's.
* Two ranks sharing cuda:0 through a gloo group (gloo all-reduces CUDA tensors): the shards of a seeded batch, equal and
  unequal, against one process running the whole batch through the unconverted model. Two runs are bit-identical, and
  a converted TripletAttention refuses before launching anything."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import _syncbn_cases as S

pytestmark = pytest.mark.gpu
DEV = "cuda"
# output / input-gradient comparison of two fused BatchNorm runs whose statistics are summed in a different order: the
# fp32 scale / shift may differ in their last bit, which moves a bf16 result across a rounding boundary (one ulp, 2^-8
# relative) here and there, and that difference travels through the following layers
BF16_RTOL = 2.0 ** -6
# per-channel quantities accumulated in fp64 / fp32 from the same values: reordering only
STAT_RTOL = 1e-6
# parameter gradients (norm-relative): every layer but the last receives its output gradient through a bf16 data gradient,
# whose elements move by one bf16 ulp where the statistics' last bit moved
GRAD_RTOL = 2.0 ** -9


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _grad_weights(name, out_shape, seed=2):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(out_shape, generator=g)


def _step(model, x, w):
    """One training step's forward and backward; returns (output, input gradient, {name: grad}, {name: buffer})."""
    x = x.clone().to(DEV).requires_grad_(True)
    out = model(x)
    out = out[:, :w.shape[1]]
    (out.float() * w.to(DEV)).sum().backward()
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
    bufs = {n: b.detach().clone() for n, b in model.named_buffers()}
    return out.detach().float().clone(), x.grad.detach().clone(), grads, bufs


def _out_shape(name, n):
    model = S.build(name).to(DEV).train()
    with torch.no_grad():
        y = model(S.inputs(name, n).to(DEV))
    return (n,) + tuple(y.shape[1:])


def _run(name, n, sync):
    model = S.build(name, sync=sync).to(DEV).train()
    w = _grad_weights(name, _out_shape(name, n))
    return _step(model, S.inputs(name, n), w)


def _assert_identical(a, b, what):
    out_a, dx_a, g_a, b_a = a
    out_b, dx_b, g_b, b_b = b
    assert torch.equal(out_a, out_b), f"{what}: output"
    assert torch.equal(dx_a, dx_b), f"{what}: input gradient"
    assert g_a.keys() == g_b.keys() and b_a.keys() == b_b.keys()
    for k in g_a:
        assert torch.equal(g_a[k], g_b[k]), f"{what}: gradient of {k}"
    for k in b_a:
        assert torch.equal(b_a[k], b_b[k]), f"{what}: buffer {k}"


@pytest.mark.parametrize("name", list(S.CASES))
def test_converted_model_is_bit_identical_without_synchronisation(name):
    plain = _run(name, 8, sync=False)
    _assert_identical(plain, _run(name, 8, sync=True), f"{name}, torch.distributed not initialised")
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{_free_port()}", rank=0, world_size=1)
    try:
        _assert_identical(plain, _run(name, 8, sync=True), f"{name}, world size 1")
    finally:
        dist.destroy_process_group()


# ------------------------------------------------------------------------------------------------------------- 2 ranks
TWO_RANK_MODELS = ["repvgg_stage", "yolov4_neck_unit", "resnet_bottleneck"]
SHARDS = {"equal": (4, 4), "unequal": (3, 5)}


def _worker(rank, port, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=2)
    torch.cuda.set_device(0)
    results = {}
    for run in ("first", "second"):
        for split, sizes in SHARDS.items():
            lo = sum(sizes[:rank])
            for name in TWO_RANK_MODELS:
                n = sum(sizes)
                x = S.inputs(name, n)[lo:lo + sizes[rank]]
                w = _grad_weights(name, _out_shape(name, n))[lo:lo + sizes[rank]]
                model = S.build(name, sync=True).to(DEV).train()
                results[(run, split, name)] = _step(model, x, w)
    # a TripletAttention whose BatchNorm would synchronise refuses before any launch
    from holocron_b200._lib import lib
    from holocron_b200.nn import TripletAttention
    att = torch.nn.SyncBatchNorm.convert_sync_batchnorm(TripletAttention()).to(DEV).train()
    before = lib().hb_launch_count()
    try:
        att(torch.randn(2, 8, 6, 6, device=DEV))
        refused = False
    except NotImplementedError:
        refused = True
    torch.cuda.synchronize()
    results["triplet"] = (refused, int(lib().hb_launch_count() - before))
    torch.save(results, os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def _close_bf16(got, ref, what):
    err = (got.double() - ref.double()).abs()
    tol = BF16_RTOL * (ref.double().abs() + ref.double().abs().mean())
    bad = err > tol
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements off, max error {float(err.max()):.3g}"


@pytest.fixture(scope="module")
def two_rank_results(tmp_path_factory):
    out = tmp_path_factory.mktemp("syncbn")
    ctx = mp.get_context("spawn")
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, port, str(out))) for r in range(2)]
    for p in procs:
        p.start()
    try:
        for p in procs:
            p.join(timeout=600)
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    return [torch.load(out / f"rank{r}.pt", weights_only=False) for r in range(2)]


@pytest.mark.parametrize("name", TWO_RANK_MODELS)
@pytest.mark.parametrize("split", list(SHARDS))
def test_two_ranks_match_the_full_batch(two_rank_results, split, name):
    what = f"{name} {split} shards"
    ref_out, ref_dx, ref_g, ref_b = _run(name, sum(SHARDS[split]), sync=False)
    ranks = [res[("first", split, name)] for res in two_rank_results]
    _close_bf16(torch.cat([r[0] for r in ranks]).to(DEV), ref_out, what + " output")
    _close_bf16(torch.cat([r[1] for r in ranks]).to(DEV), ref_dx, what + " input gradient")
    errs = {}
    for k, ref in ref_g.items():
        got = (ranks[0][2][k] + ranks[1][2][k]).to(DEV)   # parameter gradients are local sums: the ranks add up to the batch
        errs[k] = (_rel(got, ref), GRAD_RTOL)
    for k, ref in ref_b.items():
        for r, res in enumerate(ranks):
            got = res[3][k].to(DEV)
            if k.endswith("num_batches_tracked"):
                assert torch.equal(got, ref), f"{what}: rank {r} {k}"
            else:
                errs[f"rank {r} {k}"] = (_rel(got, ref), STAT_RTOL)
    bad = {k: f"{e:.3g}" for k, (e, tol) in errs.items() if not e <= tol}
    assert not bad, f"{what}: relative errors over their bounds: {bad}"


def test_two_ranks_are_deterministic(two_rank_results):
    for res in two_rank_results:
        for split in SHARDS:
            for name in TWO_RANK_MODELS:
                _assert_identical(res[("first", split, name)], res[("second", split, name)], f"{name} {split} rerun")


def test_converted_triplet_attention_refuses_in_a_two_rank_group(two_rank_results):
    for res in two_rank_results:
        refused, launches = res["triplet"]
        assert refused, "a synchronising TripletAttention ran with per-GPU statistics"
        assert launches == 0, f"{launches} kernels launched before the refusal"
