"""Times one data-parallel training step of YOLOv4 (512^2) and UNet3+ (256^2) with nn.BatchNorm2d against the same model
converted by nn.SyncBatchNorm.convert_sync_batchnorm, and counts the BatchNorm statistics all-reduces of one step.

    python -m torch.distributed.run --nproc-per-node 2 tools/syncbn_bench.py --gpus 2      # NCCL, CUDA-graph replay
    python tools/syncbn_bench.py --gpus 1     # one process: the converted model takes the plain BatchNorm path

The step is bench.py's (synthetic batch, loss, backward, one gradient all-reduce, AdaBelief), at --batch images per GPU.
Rank 0 prints one JSON line per (model, normalisation) with the GPU's name and power limit, the median and spread of the
step time over several windows of CUDA-event timing, and the statistics all-reduces per step (forward + backward)."""
import argparse
import datetime
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import holocron_b200 as hb  # noqa: E402
from bench import Workload  # noqa: E402
from holocron_b200.distributed import GradBucket, broadcast_parameters  # noqa: E402
from holocron_b200.graphs import GraphedTrainStep  # noqa: E402
from holocron_b200.nn import _fused as K  # noqa: E402
from holocron_b200.nn import functional as hbF  # noqa: E402


def run(key: str, sync: bool, batch: int, steps: int, windows: int, graph: bool, rank: int, dev) -> dict:
    wl = Workload(key)
    model = wl.model(hb, dev)
    if sync:
        model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
    broadcast_parameters(model)
    bucket = GradBucket(model.parameters())
    opt = hb.optim.AdaBelief(model.parameters(), lr=1e-3, betas=(0.95, 0.99), eps=1e-6, capturable=graph)
    devb = [t.to(dev) for t in wl.host_batch(batch, 1000 + rank)]
    devb[0] = devb[0].contiguous()

    def step(*b):
        loss = wl.loss(model, hbF, *b)
        loss.backward()
        bucket.all_reduce_mean()
        opt.step()
        bucket.zero_()
        return loss

    # statistics all-reduces of one eager step (the gradient bucket's is not one of them)
    calls = []
    real = K._all_reduce
    K._all_reduce = lambda t, group: (calls.append(t.numel()), real(t, group))[1]
    try:
        step(*devb)
    finally:
        K._all_reduce = real
    train_step = GraphedTrainStep(step, devb, warmup=3) if graph else step
    for _ in range(3):
        train_step(*devb)
    torch.cuda.synchronize()
    times = []
    for _ in range(windows):
        if dist.is_initialized():
            dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            train_step(*devb)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / steps)
    del train_step
    return {"model": f"{key} {wl.size}^2", "norm": "SyncBatchNorm" if sync else "BatchNorm2d", "batch_per_gpu": batch,
            "cuda_graph": graph, "ms_per_step_median": round(statistics.median(times), 3),
            "ms_min": round(min(times), 3), "ms_max": round(max(times), 3),
            "stat_allreduces_per_step": len(calls), "stat_allreduce_doubles_per_step": sum(calls)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--models", nargs="+", default=["yolov4", "unet3p"], choices=["yolov4", "unet3p"])
    ap.add_argument("--batch", type=int, default=16, help="images per GPU (8-16 is where synchronised statistics matter)")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--no-graph", action="store_true", help="launch the step eagerly instead of replaying a CUDA graph")
    a = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world != a.gpus:
        raise SystemExit(f"--gpus {a.gpus} but WORLD_SIZE={world}: run N > 1 under torch.distributed.run")
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev, timeout=datetime.timedelta(seconds=240))
    gpu = subprocess.run(["nvidia-smi", "-i", str(local_rank), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    for key in a.models:
        for sync in (False, True):
            res = run(key, sync, a.batch, a.steps, a.windows, not a.no_graph, rank, dev)
            if rank == 0:
                print(json.dumps({**res, "gpus": world, "gpu": gpu}), flush=True)
            torch.cuda.empty_cache()
    if world > 1:
        torch.cuda.synchronize()
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
