"""Time the Desc stage's training step on the GPU and its cylindrical convolutions layer by layer.

    python tools/train_desc_step_bench.py [--steps 20] [--out DIR]

Prints one JSON line: the median and spread of ``--steps`` C2-shaped Desc steps (512 key-points per cloud: forward, the
trainer's loss, backward, Adam; a host clock around a device synchronise), per Cylindrical_Net layer the time of each fp64
tensor-core pass (forward, dgrad, wgrad; CUDA events over 10 launches after warm-up) with its FP64 FLOP/s against the
H100 SXM data sheet's 67 TFLOP/s, the same layer on the CUDA-core bx_ts_conv_forward / bx_ts_conv_backward over an
explicitly padded copy, and the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

LAYERS = [(16, 64, 3), (64, 64, 1), (64, 128, 1), (128, 128, 1), (128, 64, 1), (64, 64, 1), (64, 32, 1), (32, 32, 1)]
DMMA_PEAK = 67e12


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:                 # noqa: BLE001
        return f"unknown ({e})"


def _time(fn, reps=10):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps * 1e-3


def layer_table(K, dev):
    from bufferx_b200 import ops
    rows = []
    for i, (Cin, Cout, Din) in enumerate(LAYERS):
        x = torch.randn((K, Cin // 4, Din * 140, 4), dtype=torch.float64, device=dev)
        Wt = torch.randn((Din * 9, Cin, Cout), dtype=torch.float64, device=dev)
        b = torch.randn(Cout, dtype=torch.float64, device=dev)
        dy = torch.randn((K, Cout // 4, 140, 4), dtype=torch.float64, device=dev)
        flop = 2.0 * K * 140 * Din * 9 * Cin * Cout
        t_f = _time(lambda: ops.cyl_forward(x, Wt, b, Din))
        t_w = _time(lambda: ops.cyl_backward(x, dy, Wt, Din, want_dx=False))
        t_fb = _time(lambda: ops.cyl_backward(x, dy, Wt, Din, want_dx=True))
        row = dict(layer=i, Cin=Cin, Cout=Cout, taps=Din * 9, fwd_ms=t_f * 1e3, wgrad_ms=t_w * 1e3, dgrad_ms=(t_fb - t_w) * 1e3,
                   fwd_tflops=flop / t_f / 1e12, wgrad_tflops=flop / t_w / 1e12, dgrad_tflops=flop / max(t_fb - t_w, 1e-9) / 1e12)
        row["fwd_share_of_67"] = row["fwd_tflops"] * 1e12 / DMMA_PEAK
        # CUDA-core route: bx_ts_conv_* (valid convolution) over an explicitly padded copy (Cin % 32 == 0 only)
        if Cin % 32 == 0:
            xp = torch.randn((K, Cin // 4, Din * 9 * 22, 4), dtype=torch.float64, device=dev)
            t_cf = _time(lambda: ops.conv_forward(xp, Wt, b, Din, 9, 22, Din, 3, 3))
            t_cb = _time(lambda: ops.conv_backward(xp, dy, Wt, Din, 9, 22, Din, 3, 3, want_dx=True))
            row.update(cuda_core_fwd_ms=t_cf * 1e3, cuda_core_bwd_ms=t_cb * 1e3)
        else:
            row.update(cuda_core_fwd_ms=None, cuda_core_bwd_ms=None)
        rows.append(row)
    return rows


def trainer_loss(out):
    """Trainer.train_epoch's Desc loss on the device (trainer.py:113-123, loss/desc_loss.py ContrastiveLoss with its
    defaults): 4 ContrastiveLoss(src_des, tgt_des, cdist(tgt_kpt, tgt_kpt)) + CrossEntropy(equi_score, gt_label)."""
    def cdist(a, b):
        return torch.sqrt(torch.sum((a[:, None] - b[None]) ** 2, dim=-1) + 1e-12)
    dist = cdist(out["src_des"], out["tgt_des"])
    dk = cdist(out["tgt_kpt"], out["tgt_kpt"]) + 10 * torch.eye(dist.shape[0], device=dist.device)
    dist = dist + 10 * (dk < 0.10).float()
    same = torch.eye(dist.shape[0], device=dist.device)
    pos = torch.max(dist * same, dim=1).values
    neg = torch.min(dist + 1e5 * same, dim=1).values
    desc = torch.mean(torch.clamp(pos - 0.1, min=0) + torch.clamp(1.4 - neg, min=0))
    return 4 * desc + torch.nn.functional.cross_entropy(out["equi_score"], out["gt_label"])


def step_times(dev, steps):
    import bufferx_b200 as bx
    from bufferx_b200.synth import add_training_clouds, init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg("C2")
    cfg.stage = "Desc"
    data = add_training_clouds(make_pair("C2", 0), cfg)
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True).to(dev)
    for p in model.Pose.parameters():
        p.requires_grad = False
    opt = torch.optim.Adam(model.get_parameter(), lr=cfg.optim.lr["Desc"], weight_decay=1e-6)
    model.train()
    times, K = [], None
    for i in range(steps + 2):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        opt.zero_grad()
        np.random.seed(i)
        out = model(data)
        trainer_loss(out).backward()
        opt.step()
        torch.cuda.synchronize()
        if i >= 2:
            times.append(time.perf_counter() - t0)
        K = int(out["src_des"].shape[0])
    return np.array(times), K


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_desc_step_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    card = _card()
    t, K = step_times(dev, a.steps)
    rows = layer_table(512, dev)
    res = dict(card=card, K=K, steps=a.steps, step_ms_median=float(np.median(t) * 1e3), step_ms_min=float(t.min() * 1e3),
               step_ms_max=float(t.max() * 1e3), layers=rows)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "train_desc_step_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
