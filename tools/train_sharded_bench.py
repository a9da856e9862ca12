"""Time sharded training steps (driver.train_step, DESIGN.md §8) on C2-shaped pairs over NCCL, one rank per GPU.

    python tools/train_sharded_bench.py [--steps 20] [--warmup 3] [--out DIR]

For every world size from 1 to the GPU count and for the Desc and the Pose stage: each rank trains its own C2 pair
(20 000 points per cloud, 512 ground-truth key-points) for --warmup + --steps steps.  Reported per (world, stage): the
median step time on rank 0 (a host clock around a device synchronise and a barrier, so the slowest rank sets it),
steps/s and pairs/s (world pairs per step), and the median time of the step's exchange (the all-gather of the record,
bx_dp_mean and the write-back of the mean) from CUDA events.  With one rank there is no collective: the exchange is
bx_dp_mean and the write-back.  The card's name and power limit are read in the same run.  Prints one JSON line.
"""
import argparse
import datetime
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def _losses():
    def desc(out):
        def cdist(a, b):
            return torch.sqrt(torch.sum((a[:, None] - b[None]) ** 2, dim=-1) + 1e-12)
        dist_ = cdist(out["src_des"], out["tgt_des"])
        dk = cdist(out["tgt_kpt"], out["tgt_kpt"]) + 10 * torch.eye(dist_.shape[0], device=dist_.device)
        dist_ = dist_ + 10 * (dk < 0.10).float()
        same = torch.eye(dist_.shape[0], device=dist_.device)
        pos = torch.max(dist_ * same, dim=1).values
        neg = torch.min(dist_ + 1e5 * same, dim=1).values
        d = torch.mean(torch.clamp(pos - 0.1, min=0) + torch.clamp(1.4 - neg, min=0))
        return 4 * d + torch.nn.functional.cross_entropy(out["equi_score"], out["gt_label"]), {}

    def pose(out):
        return torch.nn.HuberLoss()(out["pred_ind"], out["gt_ind"]), {}
    return {"Desc": desc, "Pose": pose}


def _worker(rank, world, port, steps, warmup, out):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=world, timeout=datetime.timedelta(minutes=10))
    import bufferx_b200 as bx
    from bufferx_b200 import ops
    from bufferx_b200.driver import train_step
    from bufferx_b200.synth import add_training_clouds, init_synthetic_weights, make_pair, workload_cfg
    rows = []
    for stage, loss in _losses().items():
        cfg = workload_cfg("C2")
        cfg.stage = stage
        data = add_training_clouds(make_pair("C2", rank), cfg)
        model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True)
        for p in getattr(model, "Pose" if stage == "Desc" else "Desc").parameters():
            p.requires_grad = False
        model = model.to(dev).train()
        opt = torch.optim.Adam(model.get_parameter(), lr=1e-4, weight_decay=cfg.optim.weight_decay)
        times, exch = [], []
        for i in range(warmup + steps):
            np.random.seed(i)
            ops.profiler = ops.Profiler() if i >= warmup else None
            torch.cuda.synchronize()
            dist.barrier()
            t0 = time.perf_counter()
            train_step(model, opt, data, loss)
            torch.cuda.synchronize()
            dist.barrier()
            if i >= warmup:
                times.append(time.perf_counter() - t0)
                exch.append(ops.profiler.summary()["dp_exchange"]["ms"])
        ops.profiler = None
        med = float(np.median(times))
        rows.append(dict(world=world, stage=stage, step_ms_median=med * 1e3, step_ms_min=min(times) * 1e3, step_ms_max=max(times) * 1e3,
                         steps_per_s=1.0 / med, pairs_per_s=world / med, exchange_ms_median=float(np.median(exch)),
                         record_floats=int(sum(p.numel() for p in model.parameters() if p.requires_grad) +
                                           sum(b.numel() for m in model.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm)
                                               for b in m.buffers(recurse=False)) + 1)))
    if rank == 0:
        with open(out, "w") as f:
            json.dump(rows, f)
    dist.barrier()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_sharded_bench needs CUDA devices")
    card = _card()
    results = []
    with tempfile.TemporaryDirectory() as tmp:
        for world in range(1, torch.cuda.device_count() + 1):
            path = os.path.join(tmp, f"w{world}.json")
            mp.spawn(_worker, args=(world, 29600 + world, a.steps, a.warmup, path), nprocs=world, join=True)
            with open(path) as f:
                results += json.load(f)
    line = json.dumps(dict(card=card, gpus=torch.cuda.device_count(), steps=a.steps, warmup=a.warmup, results=results))
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "train_sharded_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
