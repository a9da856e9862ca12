"""GPU experiment: per-descriptor relative error of the CUDA path against the CPU oracle, on the default conv kernel or,
with --tf32 (the convolution stacks' force_tf32), on the TF32 one.
    python tests/tools/desc_error.py C3 --tf32"""
import argparse, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import bufferx_b200 as bx
from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg
from oracle import oracle as O

ap = argparse.ArgumentParser()
ap.add_argument("workload", nargs="?", default="C2")
ap.add_argument("--tf32", action="store_true", help="run the convolution stacks on the TF32 tensor-core kernel (force_tf32)")
args = ap.parse_args()
wl = args.workload
route = "tc" if args.tf32 else "sd"
cfg = workload_cfg(wl)
cfg.match.iter_n = 2000
model = init_synthetic_weights(bx.BufferX(cfg))
sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
data = make_pair(wl, 1)
ns, nt = len(data["src_fds_pcd"]), len(data["tgt_fds_pcd"])
perms = O.draw_perms(cfg, ns, nt, 1)
model = model.cuda()
model.Desc.conv_net.force_tf32 = model.Pose.conv.force_tf32 = args.tf32
with torch.no_grad():
    model(data, perms=perms, ransac_seed=0, debug=True)
dbg = model.last_debug
_, _, _, _, _, aux = O.register_pair(sd, cfg, data, perms, 0, keep=True)
allrel = []
for i, (sc, osc) in enumerate(zip(dbg["scales"], aux["scales"])):
    for side, key in (("s", "src"), ("t", "tgt")):
        d, od = sc[side]["desc"].cpu().numpy(), osc[key]["desc"].numpy()
        x, ox = sc[side]["x"].cpu().numpy(), osc[key]["x"].numpy()
        den = np.abs(od).max(1)
        rel = np.abs(d - od).max(1) / np.where(den > 0, den, 1)
        allrel.append(rel)
        print(f"{route} {wl} scale {i} {key}: desc rel max {rel.max():.3e} p99.9 {np.quantile(rel, 0.999):.3e} median {np.median(rel):.3e} | "
              f"conv out rel {np.abs(x - ox).max() / np.abs(ox).max():.3e}")
r = np.concatenate(allrel)
print(f"ALL: max {r.max():.3e}  frac<1e-4 {(r < 1e-4).mean():.5f}  frac<5e-5 {(r < 5e-5).mean():.5f}")
