"""Wall time of one C2-shaped validation forward of the training stages (cfg.stage "Desc" / "Pose", eval mode) on the GPU.
    python tools/train_forward_bench.py [reps] [out.json]
The CPU oracle's time for the same pair and draws: tests/tools/train_forward_oracle_time.py.
GPU figure: median over `reps` forwards after two warm-up forwards, host wall clock around model(data) (the forward ends
with a host read, so the clock covers the device work)."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bufferx_b200 as bx  # noqa: E402
from bufferx_b200.synth import add_training_clouds, init_synthetic_weights, make_pair, workload_cfg  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
res = dict(gpu=torch.cuda.get_device_name(0), workload="C2", pos_num=None)
for stage in ("Desc", "Pose"):
    cfg = workload_cfg("C2")
    cfg.stage = stage
    res["pos_num"] = cfg.train.pos_num
    data = add_training_clouds(make_pair("C2", 0), cfg)
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True).cuda()
    ts = []
    with torch.no_grad():
        for r in range(reps + 2):
            np.random.seed(r)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = model(data)
            torch.cuda.synchronize()
            if r >= 2:
                ts.append(time.perf_counter() - t0)
    res[stage] = dict(gpu_ms_median=1e3 * float(np.median(ts)), gpu_ms_min=1e3 * float(np.min(ts)),
                      sds_points=[len(data["src_sds_pcd"]), len(data["tgt_sds_pcd"])])
print(json.dumps(res))
if len(sys.argv) > 2:
    os.makedirs(os.path.dirname(os.path.abspath(sys.argv[2])), exist_ok=True)
    with open(sys.argv[2], "w") as f:
        json.dump(res, f)
