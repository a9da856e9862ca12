"""CPU oracle time of the C2-shaped validation forward that tools/train_forward_bench.py times on the GPU.
    python tests/tools/train_forward_oracle_time.py [out.json]"""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import bufferx_b200 as bx  # noqa: E402
from bufferx_b200.synth import add_training_clouds, init_synthetic_weights, make_pair, workload_cfg  # noqa: E402
from oracle import train_stages as TS  # noqa: E402

res = dict(workload="C2", cpu_threads=torch.get_num_threads(), host_cpus=os.cpu_count())
for stage in ("Desc", "Pose"):
    cfg = workload_cfg("C2")
    cfg.stage = stage
    data = add_training_clouds(make_pair("C2", 0), cfg)
    sd = {k: v.detach().clone() for k, v in init_synthetic_weights(bx.BufferX(cfg), trained_pose=True).state_dict().items()}
    TS.O.build()
    np.random.seed(0)
    t0 = time.perf_counter()
    TS.train_forward(stage, sd, cfg, data)
    res[stage] = dict(cpu_oracle_s=time.perf_counter() - t0)
print(json.dumps(res))
if len(sys.argv) > 1:
    with open(sys.argv[1], "w") as f:
        json.dump(res, f)
