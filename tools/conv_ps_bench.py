"""GPU experiment: the descriptor conv stack (Cylindrical_Net on K patches), conv_sd_kernel against the per-sample kernel
(bx_conv_ps.cu), layer by layer on the same card, the two kernels alternating within every repetition.
    python tools/conv_ps_bench.py [K] [reps]       # per-layer us and fp32-equivalent TFLOP/s of both, and the ratio
Each layer of each kernel reads the same input (the previous layer's output of conv_sd_kernel) and writes into a zeroed
buffer; its output bytes are compared with conv_sd_kernel's.  The production stack runs the last layer (fp32 output) on
conv_sd_kernel; it is timed here on both."""
import json, os, subprocess, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bufferx_b200 as bx
from bufferx_b200 import ops
from bufferx_b200.synth import init_synthetic_weights, workload_cfg

K = int(sys.argv[1]) if len(sys.argv) > 1 else 9000
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 20
dev = torch.device("cuda")
L = init_synthetic_weights(bx.BufferX(workload_cfg("C2"))).cuda().Desc.conv_net.folded()
torch.manual_seed(0)
x = ops.sd_pack(torch.relu(torch.randn(K, 48, 7, 20, device=dev)))        # the presplit image bx_spt_pnt_sd writes
outs = {k: [ops.conv_sd_buffer(K, l["cout"], dev).zero_() if i < len(L) - 1 else torch.zeros((K, l["cout"] // 4, 140, 4), device=dev)
            for i, l in enumerate(L)] for k in ("sd", "ps")}
ins = [x] + outs["sd"][:-1]
fn = {"sd": ops.conv_layer_sd, "ps": ops.conv_layer_ps}
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
times = {k: [[] for _ in L] for k in fn}
for r in range(reps + 2):
    for k in (("sd", "ps") if r % 2 == 0 else ("ps", "sd")):
        for i, l in enumerate(L):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn[k](ops.GEOM_CYL3D if i == 0 else ops.GEOM_CYL2D, ins[i], l["w_sd"], l["b"], outs[k][i], K, l["cin"], l["cout"], l["relu"])
            b.record()
            if r >= 2:
                times[k][i].append((a, b))
torch.cuda.synchronize()
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
rows, tot = [], {"sd": 0.0, "ps": 0.0}
for i, l in enumerate(L):
    fl = 2.0 * K * 140 * l["cin"] * l["cout"] * (27 if i == 0 else 9)
    med = {}
    for k in fn:
        ts = sorted(a.elapsed_time(b) for a, b in times[k][i])
        med[k] = ts[len(ts) // 2]
        tot[k] += med[k]
    same = torch.equal(outs["sd"][i].view(torch.int16 if i < len(L) - 1 else torch.int32), outs["ps"][i].view(torch.int16 if i < len(L) - 1 else torch.int32))
    rows.append(dict(layer=i, cin=l["cin"], cout=l["cout"], sd_us=med["sd"] * 1e3, ps_us=med["ps"] * 1e3, speedup=med["sd"] / med["ps"],
                     sd_tflops=fl / med["sd"] / 1e9, ps_tflops=fl / med["ps"] / 1e9, bit_identical=same))
    print(f"L{i}: {l['cin']:3d}->{l['cout']:3d}  sd {med['sd'] * 1e3:7.1f} us  ps {med['ps'] * 1e3:7.1f} us  x{med['sd'] / med['ps']:.3f}  identical={same}")
print(f"stack: sd {tot['sd'] * 1e3:.1f} us  ps {tot['ps'] * 1e3:.1f} us  x{tot['sd'] / tot['ps']:.3f}   [{smi}, K={K}, median of {reps}]")
print(json.dumps(dict(gpu=smi, K=K, reps=reps, layers=rows, stack_sd_us=tot["sd"] * 1e3, stack_ps_us=tot["ps"] * 1e3)))
