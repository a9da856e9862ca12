"""CPU time of the float64 ICP test oracle (oracle/icp_fp64.py, NumPy/scipy -- not Open3D) on the pairs tools/icp_bench.py
times on the GPU (synth.kitti_icp_pair, r = 0.20, init = I, max_iteration = 200).
    python tests/tools/icp_oracle_time.py [--seeds 0 1]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bufferx_b200  # noqa: E402,F401
from bufferx_b200.synth import kitti_icp_pair  # noqa: E402
from oracle.icp_fp64 import icp_fp64  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--seeds", type=int, nargs="+", default=[0, 1])
a = ap.parse_args()
rows = []
for seed in a.seeds:
    src, tgt = kitti_icp_pair(seed)
    t0 = time.perf_counter()
    out = icp_fp64(src, tgt, 0.20, max_iteration=200)
    rows.append(dict(seed=seed, oracle_fp64_cpu_s=round(time.perf_counter() - t0, 3), iterations=out["iterations"],
                     fitness=round(out["fitness"], 6), rmse=round(out["rmse"], 6)))
print(json.dumps(dict(tool="icp_oracle_time", host_cpus=os.cpu_count(), pairs=rows,
                      note="the NumPy/scipy float64 test oracle on the host CPU, not Open3D")))
