"""Point-to-point ICP at the KITTI loader's call shape (r = 0.20, init = I, max_iteration = 200) on C3-sized synthetic scan
pairs (synth.kitti_icp_pair: 2 x 120 000 points, pre-aligned by a perturbed ground truth), from CUDA events after warm-up:
  gpu_ms_per_call        the call as the loader makes it (max_iteration = 200): the target grid, the live iterations, the
                         3 x (200 - iterations) launches queued after the stop that return at once, and ops.icp's
                         workspace allocation (from torch's caching allocator);
  gpu_ms_live            the same call with max_iteration = the iterations the run needs, so nothing is queued after it;
  gpu_ms_tail            gpu_ms_per_call - gpu_ms_live: the cost of the no-op steps after the stop;
  gpu_ms_per_iteration   gpu_ms_live / iterations (still including the one-off grid build and first evaluation).
The card's name and power limit are read in the same run.  The CPU time of the float64
test oracle on the same pairs (not Open3D, which is not measured) comes from tests/tools/icp_oracle_time.py: nothing under
tools/ imports the oracle.

    python tools/icp_bench.py [--seeds 0 1] [--reps 5]

Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception as e:   # the measurement still stands; the card is then unknown
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seeds", type=int, nargs="+", default=[0, 1])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()

    import numpy as np
    import torch

    import bufferx_b200 as bx
    from bufferx_b200.synth import kitti_icp_pair

    assert torch.cuda.is_available(), "icp_bench needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    rows = []
    for seed in a.seeds:
        s_np, t_np = kitti_icp_pair(seed)
        src = torch.from_numpy(s_np).to(dev)
        tgt = torch.from_numpy(t_np).to(dev)
        init = torch.eye(4, dtype=torch.float64, device=dev)
        def timed(max_iteration):
            run = lambda: bx.ops.icp(src, tgt, 0.20, init, 1e-6, 1e-6, max_iteration)
            for _ in range(2):
                res, _ = run()
            torch.cuda.synchronize()
            times = []
            for _ in range(a.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                res, _ = run()
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
            return res, times

        res, times = timed(200)
        T, fit, rmse, ncorr, iters, conv = bx.ops.decode_icp_result(res.cpu())
        res_live, times_live = timed(iters)
        assert bx.ops.decode_icp_result(res_live.cpu())[4] == iters
        ms, ms_live = float(np.median(times)), float(np.median(times_live))
        row = dict(seed=seed, n_src=int(src.shape[0]), n_tgt=int(tgt.shape[0]), iterations=iters, converged=conv,
                   gpu_ms_per_call=round(ms, 3), gpu_ms_spread=[round(min(times), 3), round(max(times), 3)],
                   gpu_ms_live=round(ms_live, 3), gpu_ms_live_spread=[round(min(times_live), 3), round(max(times_live), 3)],
                   gpu_ms_tail=round(ms - ms_live, 3), gpu_ms_per_iteration=round(ms_live / max(iters, 1), 4),
                   fitness=round(fit, 6), rmse=round(rmse, 6))
        rows.append(row)
    print(json.dumps(dict(tool="icp_bench", card=card(), call="r=0.20 init=I max_iteration=200", pairs=rows)))


if __name__ == "__main__":
    main()
