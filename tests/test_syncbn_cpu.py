"""nn.SyncBatchNorm on the fused BatchNorm path, host side (no CUDA kernels): converted model trees keep their
checkpoints, every unit recogniser routes a SyncBatchNorm where it routes a BatchNorm2d, the "synchronise or not"
decision, the fp64 buffers the statistics all-reduces act on, and the refusal of a synchronising TripletAttention."""
import importlib
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from torch import nn

from holocron_b200 import models
from holocron_b200.models.classification import mobileone as mobileone_mod
from holocron_b200.nn import TripletAttention
from holocron_b200.nn import _fused as K
from holocron_b200.trainer import freeze_bn

import _syncbn_cases as S


@pytest.mark.parametrize("arch", ["repvgg_a0", "rexnet1_0x", "yolov4", "unet3p"])
def test_converted_trees_keep_state_dict_keys(arch):
    torch.manual_seed(0)
    model = getattr(models, arch)()
    keys = list(model.state_dict())
    conv = nn.SyncBatchNorm.convert_sync_batchnorm(model)
    assert list(conv.state_dict()) == keys
    assert not any(isinstance(m, nn.BatchNorm2d) for m in conv.modules())
    assert any(isinstance(m, nn.SyncBatchNorm) for m in conv.modules())


def test_is_batch_norm():
    assert K.is_batch_norm(nn.BatchNorm2d(8)) and K.is_batch_norm(nn.SyncBatchNorm(8))
    assert not K.is_batch_norm(nn.GroupNorm(2, 8)) and not K.is_batch_norm(nn.LayerNorm(8))


class _Recorder:
    """Stands in for the fused functions: records the normalisation layers they receive, returns a fake activation."""

    def __init__(self, monkeypatch):
        self.bns = []

        def bn_act(us, bns, *a, **k):
            self.bns.extend(bns)
            return us[0]

        def repblock(x, w3, w1, bns, *a, **k):
            self.bns.extend(bns)
            return torch.zeros(x.shape[0], w3.shape[0], x.shape[2] // a[0], x.shape[3] // a[0])

        def conv2d(x, weight, bias=None, stride=1, padding=0, *a, **k):
            return torch.zeros(x.shape[0], weight.shape[0], x.shape[2] // stride, x.shape[3] // stride)

        monkeypatch.setattr(K, "bn_act", bn_act)
        monkeypatch.setattr(K, "repblock", repblock)
        monkeypatch.setattr(K, "conv2d", conv2d)
        monkeypatch.setattr(K, "to_channels_last_bf16", lambda x, c=None: x)


@pytest.mark.parametrize("name", ["repvgg_stage", "yolov4_neck_unit", "resnet_bottleneck", "mobileone"])
def test_sync_batchnorm_is_routed_like_batchnorm(monkeypatch, name):
    """Every BatchNorm of the piece reaches a fused function, converted or not (CPU tensors flow through the recording
    stand-ins; the real functions refuse them)."""
    rec = _Recorder(monkeypatch)
    monkeypatch.setattr(mobileone_mod, "_fusable", lambda branches, x: True)
    import holocron_b200.nn._dwconv as dw
    monkeypatch.setattr(dw, "dwconv2d", lambda x, w, b, s, p: x[:, :, ::s, ::s])
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    seen = []
    for sync in (False, True):
        rec.bns.clear()
        model = S.build(name, sync=sync).train()
        model(S.inputs(name, 2))
        seen.append([type(b).__name__ for b in rec.bns])
    n = sum(isinstance(m, nn.BatchNorm2d) for m in S.build(name).modules())
    assert seen[0] == ["BatchNorm2d"] * n
    assert seen[1] == ["SyncBatchNorm"] * n


def test_unet_skip_batchnorm_is_routed(monkeypatch):
    """DynamicUNet's decoder block normalises its skip features on the fused pass, converted or not."""
    unet = importlib.import_module("holocron_b200.models.segmentation.unet")
    calls = []
    monkeypatch.setattr(unet, "run_fused", lambda mods, x, *a, **k: calls.append(mods) or x)
    block = nn.SyncBatchNorm.convert_sync_batchnorm(unet.UBlock(8, 16, 8))
    block.upsample = nn.Sequential(nn.Conv2d(16, 64, 1), nn.PixelShuffle(2))
    block.block = nn.Identity()
    block(torch.randn(1, 8, 8, 8), torch.randn(1, 16, 4, 4))
    assert len(calls) == 1 and isinstance(calls[0][0], nn.SyncBatchNorm)


# --------------------------------------------------------------------------------------------- synchronise or not
def test_no_synchronisation_without_an_initialised_group():
    bn = nn.SyncBatchNorm(8).train()
    assert not dist.is_initialized()
    assert K.sync_group([bn], True) is None
    assert K.sync_group([nn.BatchNorm2d(8)], True) is None


def test_no_synchronisation_at_world_size_one():
    port = _free_port()
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    try:
        assert K.sync_group([nn.SyncBatchNorm(8).train()], True) is None
    finally:
        dist.destroy_process_group()


def test_sync_buffer_layout():
    nb, c = 3, 40
    sums = K.sync_sums_buffer(nb, c, "cpu")
    assert sums.dtype == torch.float64 and sums.numel() == nb * c * 2 + 1
    cnt = K.sync_count(sums)
    assert cnt.numel() == 1 and cnt.data_ptr() == sums.data_ptr() + 8 * nb * c * 2
    scratch = torch.zeros(1000, dtype=torch.float64)
    head = K.sync_grad_sums(scratch, nb, c)
    assert head.numel() == (1 + nb) * c and head.data_ptr() == scratch.data_ptr() and head.is_contiguous()


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, port, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=2)
    res = {}
    bn = nn.SyncBatchNorm(8)
    res["train"] = K.sync_group([bn.train()], True) is not None
    res["eval"] = K.sync_group([bn.eval()], bn.training) is None
    frozen = nn.SyncBatchNorm(8)
    for p in frozen.parameters():
        p.requires_grad_(False)
    freeze_bn(nn.Sequential(frozen).train())
    res["frozen"] = K.sync_group([frozen], frozen.training) is None
    res["plain"] = K.sync_group([nn.BatchNorm2d(8).train()], True) is None
    try:
        K.sync_group([nn.SyncBatchNorm(8).train(), nn.BatchNorm2d(8).train()], True)
        res["mixed"] = False
    except NotImplementedError:
        res["mixed"] = True
    # forward buffer: rank r packs (sum, sum of squares) of its rows and its row count; after the all-reduce every rank
    # unpacks the global sums and count
    nb, c = 2, 8
    rows = [torch.arange(6 * 2 * c, dtype=torch.float64).view(6, 2, c) / 7, torch.linspace(-2, 3, 9 * 2 * c,
            dtype=torch.float64).view(9, 2, c)]
    mine = rows[rank]
    sums = K.sync_sums_buffer(nb, c, "cpu")
    body = sums[:-1].view(nb, c, 2)
    body[..., 0] = mine.sum(0)
    body[..., 1] = (mine * mine).sum(0)
    K.sync_count(sums).fill_(mine.shape[0])
    K._all_reduce(sums, K.sync_group([bn.train()], True))
    full = torch.cat(rows)
    res["fwd"] = (torch.allclose(body[..., 0], full.sum(0), rtol=1e-15, atol=0)
                  and torch.allclose(body[..., 1], (full * full).sum(0), rtol=1e-15, atol=0)
                  and float(K.sync_count(sums)) == 15)
    # backward: only the [1 + nb][c] head of the scratch travels, the per-block partials behind it stay local
    scratch = torch.full((200,), float(rank + 1), dtype=torch.float64)
    K._all_reduce(K.sync_grad_sums(scratch, nb, c), K.sync_group([bn.train()], True))
    res["bwd"] = bool((scratch[:(1 + nb) * c] == 3).all()) and bool((scratch[(1 + nb) * c:] == rank + 1).all())
    # TripletAttention converted: refuses before it looks at the device (a CPU tensor here)
    att = nn.SyncBatchNorm.convert_sync_batchnorm(TripletAttention()).train()
    try:
        att(torch.randn(2, 8, 6, 6))
        res["triplet"] = "ran"
    except NotImplementedError as e:
        res["triplet"] = "SyncBatchNorm" in str(e)
    except Exception as e:   # noqa: BLE001 - any other refusal (the device check) is the failure being tested for
        res["triplet"] = repr(e)
    torch.save(res, os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_gloo_group(tmp_path):
    ctx = mp.get_context("spawn")
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, port, str(tmp_path))) for r in range(2)]
    for p in procs:
        p.start()
    try:
        for p in procs:
            p.join(timeout=180)
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    for r in range(2):
        res = torch.load(tmp_path / f"rank{r}.pt")
        assert res == {"train": True, "eval": True, "frozen": True, "plain": True, "mixed": True, "fwd": True,
                       "bwd": True, "triplet": True}, (r, res)
