"""FPS of clouds beyond one cluster's registers (bx_fps_large) against the largest cluster tier, from CUDA events after
warm-up (median and spread of --reps timed calls, each bracketed by a device synchronise):
  fps_large_ms   ops.fps_large at N = 524289, 1048576 and 1638400 (synthetic C3 clouds), npoint 2000, including the
                 workspace allocation and the counter reset;
  fps_t512x64_ms ops.fps at N = 524288 (bx_fps's T512x64 tier, one 16-CTA cluster), npoint 2000, for comparison;
  forward_ms     one eager BufferX.forward of a C3 pair of 700000 / 600000 points (the C3 configuration, 2048 key points,
                 3 scales, no early exit), host clock around a call that ends in its device-to-host read.
The card's name and power limit are read in the same run.

    python tools/fps_large_bench.py [--reps 20] [--forward-reps 3]

Prints one JSON line.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from icp_bench import card  # noqa: E402


def _events(run, reps, warmup=3):
    import numpy as np
    import torch
    for _ in range(warmup):
        run()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return dict(median=round(float(np.median(times)), 3), spread=[round(min(times), 3), round(max(times), 3)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--forward-reps", type=int, default=3)
    ap.add_argument("--npoint", type=int, default=2000)
    a = ap.parse_args()

    import numpy as np
    import torch

    import bufferx_b200 as bx
    from bufferx_b200 import ops
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg

    assert torch.cuda.is_available(), "fps_large_bench needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    out = dict(tool="fps_large_bench", card=card(), npoint=a.npoint, fps_large_ms={})
    for n in (524289, 1048576, ops.FPS_LARGE_MAX_POINTS):
        x = torch.from_numpy(make_pair("C3", 7, n_src=n, n_tgt=1000)["src_fds_pcd"]).to(dev)
        out["fps_large_ms"][str(n)] = _events(lambda: ops.fps_large(x, a.npoint), a.reps)
    x = torch.from_numpy(make_pair("C3", 7, n_src=524288, n_tgt=1000)["src_fds_pcd"]).to(dev)
    out["fps_t512x64_ms"] = {"524288": _events(lambda: ops.fps(x, [0, 524288], a.npoint), a.reps)}

    cfg = workload_cfg("C3")
    cfg.match.enable_early_exit = False
    model = init_synthetic_weights(bx.BufferX(cfg)).to(dev).eval()
    data = make_pair("C3", 11, n_src=700000, n_tgt=600000)
    times = []
    with torch.no_grad():
        model(data)                                   # warm-up: kernel attributes, allocator
        for _ in range(a.forward_reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model(data)                               # ends in the pair's device-to-host read
            times.append((time.perf_counter() - t0) * 1e3)
    out["forward_ms"] = {"700000/600000": dict(median=round(float(np.median(times)), 2), spread=[round(min(times), 2), round(max(times), 2)])}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
