"""GPU timing of the drop-in modules under dropin/ at the BUFFER-X reference's call shapes.

    python tools/dropin_bench.py [--iters N] [--json OUT]

Each op is warmed up, then timed over --iters calls between two CUDA events on the current stream (mean per call).  The
card name and power limit are read in the same run and printed with the numbers.  Shapes:
    furthest_point_sample  B=1, N=20000, npoint=1500                                   (BUFFERX.py:338-339)
    gather_operation       B=1, C=3, N=20000, M=1500                                   (BUFFERX.py:342-345)
    ball_query             B=1, N=20000, M=1500, nsample=512, the C2 radius             (patch_embedder.py:99)
    grouping_operation     B=1, C=3, N=20000, M=1500, S=512                            (patch_embedder.py:101)
    ball_query             B=1500, N=512, M=420, nsample=10, voxel radius 0.8/3         (common.py:442, sphere_query)
    grouping_operation     B=1500, C=3, N=512, M=420, S=10                             (common.py:453)
    KNN(k=1)               B=1, Nr=Nq=1500, D=32 (mutual matching, BUFFERX.py:481,486)
    KNN(k=1)               B=1, Nr=Nq=20000, D=3 (ground-truth matches, BUFFERX.py:511)
    svd                    B=1500 3x3 covariances (cal_Z_axis, common.py:715)
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "dropin"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name()


def timed(fn, iters, warmup=5):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "dropin_bench needs a CUDA device"
    import knn_cuda
    import torch_batch_svd
    from pointnet2_ops import pointnet2_utils as p2
    from bufferx_b200.synth import make_pair
    from bufferx_b200.models.patch_embedder import voxel_table

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    pts = torch.from_numpy(make_pair("C2", 0)["src_fds_pcd"].astype(np.float32)).to(dev)[None].contiguous()
    r = float(np.float32(np.load(os.path.join(ROOT, "tests", "golden", "c2_seed0.npz"))["des_r"][0]))
    fps_idx = p2.furthest_point_sample(pts, 1500)
    pts_t = pts.transpose(1, 2).contiguous()
    kpts = p2.gather_operation(pts_t, fps_idx).transpose(1, 2).contiguous()
    big_idx = p2.ball_query(r, 512, pts, kpts)
    patches = p2.grouping_operation(pts_t, big_idx).permute(0, 2, 3, 1)[0].contiguous()      # [1500, 512, 3]
    local = patches - patches[:, -1:, :]
    delta = (local / r).contiguous()
    vox = torch.from_numpy(voxel_table(3, 20, 7)).to(dev)[None].expand(1500, -1, -1).contiguous()
    small_idx = p2.ball_query(0.8 / 3, 10, delta, vox)
    delta_t = delta.transpose(1, 2).contiguous()
    desc = torch.randn((1, 1500, 32), device=dev)
    desc2 = torch.randn((1, 1500, 32), device=dev)
    knn = knn_cuda.KNN(k=1, transpose_mode=True)
    cov = torch.matmul(local.transpose(1, 2), local)
    pts2 = pts + 0.01 * torch.randn_like(pts)

    rows = [
        ("furthest_point_sample B=1 N=20000 npoint=1500", lambda: p2.furthest_point_sample(pts, 1500)),
        ("gather_operation B=1 C=3 N=20000 M=1500", lambda: p2.gather_operation(pts_t, fps_idx)),
        ("ball_query B=1 N=20000 M=1500 nsample=512", lambda: p2.ball_query(r, 512, pts, kpts)),
        ("grouping_operation B=1 C=3 N=20000 M=1500 S=512", lambda: p2.grouping_operation(pts_t, big_idx)),
        ("ball_query B=1500 N=512 M=420 nsample=10", lambda: p2.ball_query(0.8 / 3, 10, delta, vox)),
        ("grouping_operation B=1500 C=3 N=512 M=420 S=10", lambda: p2.grouping_operation(delta_t, small_idx)),
        ("KNN k=1 B=1 Nr=Nq=1500 D=32", lambda: knn(desc, desc2)),
        ("KNN k=1 B=1 Nr=Nq=20000 D=3", lambda: knn(pts, pts2)),
        ("svd B=1500 3x3", lambda: torch_batch_svd.svd(cov)),
    ]
    gpu = card()
    out = {"gpu": gpu, "iters": args.iters, "ms": {}}
    print(f"GPU: {gpu}")
    for name, fn in rows:
        ms = timed(fn, args.iters)
        out["ms"][name] = ms
        print(f"{name:52s} {ms * 1e3:10.1f} us")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
