"""GPU experiment: the descriptor conv stack alone (Cylindrical_Net on K patches), per-layer CUDA-event times.
    python tools/conv_bench.py [K] [reps] [--tf32]  # prints per-layer ms and TFLOP/s (fp32-equivalent)
--tf32 sets the stack's force_tf32, its fall-back to the TF32 tensor-core kernel, instead of the shifted-descriptor
fp16-split kernel.
Under ncu:  ncu --set full -k regex:conv_tc --launch-skip 16 -c 8 python tools/conv_bench.py 1500 3 --tf32"""
import argparse, os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bufferx_b200 as bx
from bufferx_b200 import ops
from bufferx_b200.synth import init_synthetic_weights, workload_cfg

ap = argparse.ArgumentParser()
ap.add_argument("K", type=int, nargs="?", default=1500)
ap.add_argument("reps", type=int, nargs="?", default=10)
ap.add_argument("--tf32", action="store_true", help="run the stack on the TF32 tensor-core kernel (force_tf32)")
args = ap.parse_args()
K, reps = args.K, args.reps
cfg = workload_cfg("C2")
model = init_synthetic_weights(bx.BufferX(cfg)).cuda()
net = model.Desc.conv_net
net.force_tf32 = args.tf32
MODE = "tc" if net.force_tf32 else "sd"
L = net.folded()
dev = torch.device("cuda")
torch.manual_seed(0)
x = torch.relu(torch.randn(K, 4, 420, 4, device=dev))            # channel-blocked
if MODE == "sd":     # production feeds the first layer the presplit image written by bx_spt_pnt_sd
    x = ops.sd_pack(ops.from_blocked(x).view(K, 16, 3, 140).permute(0, 2, 1, 3).reshape(K, 48, 7, 20))
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
if MODE == "sd":     # layer-to-layer activations in the presplit padded fp16 format, fp32 out of the last layer
    bufs = [ops.conv_sd_buffer(K, l["cout"], dev) if i < len(L) - 1 else torch.empty((K, l["cout"] // 4, 140, 4), device=dev) for i, l in enumerate(L)]
else:
    bufs = [torch.empty((K, l["cout"] // 4, 140, 4), device=dev) for l in L]
times = [[] for _ in L]
for r in range(reps + 2):
    flush.zero_()
    cur = x
    for i, l in enumerate(L):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        if MODE == "sd":
            ops.conv_layer_sd(ops.GEOM_CYL3D if i == 0 else ops.GEOM_CYL2D, cur, l["w_sd"], l["b"], bufs[i], K, l["cin"], l["cout"], l["relu"], None)
        elif i == 0:
            ops.conv_layer_tc(ops.GEOM_CYL3D, cur, l["w_tc"], l["b"], bufs[i], K, l["cin"], l["cout"], 3, 7, 20, 3, 3, 3, l["relu"])
        else:
            ops.conv_layer_tc(ops.GEOM_CYL2D, cur, l["w_tc"], l["b"], bufs[i], K, l["cin"], l["cout"], 1, 7, 20, 1, 3, 3, l["relu"])
        b.record()
        cur = bufs[i]
        if r >= 2:
            times[i].append((a, b))
torch.cuda.synchronize()
tot_ms, tot_fl = 0.0, 0.0
for i, l in enumerate(L):
    ms = sum(a.elapsed_time(b) for a, b in times[i]) / len(times[i])
    taps = l["k"][0] * l["k"][1] * l["k"][2]
    fl = 2.0 * K * 140 * l["cin"] * l["cout"] * taps
    stages = l["cin"] // 16 * taps
    tot_ms += ms
    tot_fl += fl
    print(f"L{i}: {l['cin']:3d}->{l['cout']:3d} taps {taps:2d} stages {stages:3d}  {ms * 1e3:7.1f} us  {fl / ms / 1e9:6.1f} TFLOP/s")
print(f"[{MODE}] stack: {tot_ms * 1e3:.1f} us  {tot_fl / tot_ms / 1e9:.1f} TFLOP/s fp32-equivalent")
