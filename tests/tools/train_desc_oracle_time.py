"""Time the float64 CPU oracle of the Desc stage's training step (oracle/train_desc.py: forward, the trainer's loss,
backward) on the C2 pair tools/train_desc_step_bench.py times on the GPU (512 matched key-points).  Prints one JSON line."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import oracle as O  # noqa: E402
from oracle import train_desc as TD  # noqa: E402
from oracle.train_step import bn_hparams  # noqa: E402


def main():
    import bufferx_b200 as bx
    from bufferx_b200.synth import add_training_clouds, init_synthetic_weights, make_pair, workload_cfg
    O.build()
    cfg = workload_cfg("C2")
    cfg.stage = "Desc"
    data = add_training_clouds(make_pair("C2", 0), cfg)
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    np.random.seed(0)
    t0 = time.perf_counter()
    r = TD.train_step(sd, bn_hparams(model), cfg, data)
    TD.desc_loss(r["src_des"], r["tgt_des"], r["tgt_kpt"], r["equi_score"], r["gt_label"]).backward()
    print(json.dumps(dict(oracle_fp64_cpu_s=time.perf_counter() - t0, oracle_keypoints=int(r["K"]),
                          oracle_torch_threads=torch.get_num_threads(), oracle_cpus=os.cpu_count())))


if __name__ == "__main__":
    main()
