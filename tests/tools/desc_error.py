"""GPU experiment: per-descriptor relative error of the CUDA path against the CPU oracle, on the default conv kernel or,
with BX_CONV=tc, on the TF32 one.
    BX_CONV=tc python tests/tools/desc_error.py C3"""
import os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import bufferx_b200 as bx
from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg
from oracle import oracle as O

wl = sys.argv[1] if len(sys.argv) > 1 else "C2"
cfg = workload_cfg(wl)
cfg.match.iter_n = 2000
model = init_synthetic_weights(bx.BufferX(cfg))
sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
data = make_pair(wl, 1)
ns, nt = len(data["src_fds_pcd"]), len(data["tgt_fds_pcd"])
perms = O.draw_perms(cfg, ns, nt, 1)
model = model.cuda()
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
        print(f"{os.environ.get('BX_CONV','tc')} {wl} scale {i} {key}: desc rel max {rel.max():.3e} p99.9 {np.quantile(rel, 0.999):.3e} median {np.median(rel):.3e} | "
              f"conv out rel {np.abs(x - ox).max() / np.abs(ox).max():.3e}")
r = np.concatenate(allrel)
print(f"ALL: max {r.max():.3e}  frac<1e-4 {(r < 1e-4).mean():.5f}  frac<5e-5 {(r < 5e-5).mean():.5f}")
