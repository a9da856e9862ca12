"""GPU experiment: FPS latency of one pair's key-point sampling (both clouds in one launch), C2 (2 x 20000 points, 2000
samples) and C3 (2048 samples).
    python tools/fps_bench.py"""
import os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bufferx_b200 import ops
from bufferx_b200.synth import make_pair
for wl, m in (("C2", 2000), ("C3", 2048)):
    d = make_pair(wl, 0)
    ns, nt = len(d["src_fds_pcd"]), len(d["tgt_fds_pcd"])
    xyz = torch.from_numpy(np.concatenate([d["src_fds_pcd"], d["tgt_fds_pcd"]])).cuda()
    for _ in range(3):
        ops.fps(xyz, [0, ns, ns + nt], m)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(10):
        ops.fps(xyz, [0, ns, ns + nt], m)
    b.record(); b.synchronize()
    ms = a.elapsed_time(b) / 10
    print(f"{wl} ({ns}+{nt} pts, {m} samples) {ms:7.3f} ms  {1e3 * ms / m:6.3f} us/iteration")
