"""Time one C2-shaped Pose-stage training step on the GPU: 512 matched key-points, model.train() with Desc frozen, the
forward (both descriptor calls with batch statistics, CostNet), HuberLoss, backward and the Adam step, as
Trainer.train_epoch takes it (trainer.py:93-167).  Prints one JSON line: the median and spread of --runs timed steps (host
clock around a device synchronise), the card's name and power limit read in the same run, and the time of the float64 CPU
oracle on the same pair (tests/tools/train_step_oracle_time.py, run as a separate process).

    python tools/train_step_bench.py [--runs 20] [--warmup 3] [--no-oracle]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_step_bench needs a CUDA device")
    import bufferx_b200 as bx
    from bufferx_b200.synth import add_training_clouds, init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg("C2")
    cfg.stage = "Pose"
    data = add_training_clouds(make_pair("C2", 0), cfg)
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model = model.cuda()
    for p in model.Desc.parameters():
        p.requires_grad = False
    opt = torch.optim.Adam(model.get_parameter(), lr=1e-4, weight_decay=1e-6)
    huber = torch.nn.HuberLoss()
    model.train()
    times, K = [], None
    for i in range(a.warmup + a.runs):
        np.random.seed(i)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        opt.zero_grad()
        out = model(data)
        loss = huber(out["pred_ind"], out["gt_ind"].float())
        loss.backward()
        opt.step()
        torch.cuda.synchronize()
        if i >= a.warmup:
            times.append(time.perf_counter() - t0)
        K = out["pred_ind"].shape[0]
    res = dict(metric="pose_train_step", workload="C2", keypoints=int(K), runs=a.runs, gpu=gpu_info(),
               step_ms_median=1e3 * float(np.median(times)), step_ms_min=1e3 * float(np.min(times)),
               step_ms_max=1e3 * float(np.max(times)))
    if not a.no_oracle:          # the float64 CPU oracle on the same pair, in its own process
        q = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "tools", "train_step_oracle_time.py")], capture_output=True,
                           text=True, cwd=ROOT)
        if q.returncode != 0:
            raise SystemExit("oracle timing failed:\n" + q.stderr[-2000:])
        res.update(json.loads(q.stdout.strip().splitlines()[-1]))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
