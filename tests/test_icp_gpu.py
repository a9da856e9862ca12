"""GPU point-to-point ICP (csrc/bx_icp.cu, bufferx_b200.registration) against the float64 oracle (oracle/icp_fp64.py).

Every case runs on the GPU once per step k (max_iteration = k) and once in full.  Step k is checked against the oracle's
step k with oracle/icp_cases.check_step: where no decision is within reach of the measured perturbation the correspondence
set and fitness are equal and rmse is within the derived bound; where some are (exact ties, points at r), the run is held to
the bounds for m marginal points from that step on.  Where the fit is unique, the GPU's transformation at every checked step
must first lie within the a-priori bound computed from the oracle's Sigmas (icp_cases.t_bound), and the decisions are
classified with that bound, not with the measured difference.  The full run must stop after as many updates as the oracle
and its transformation is held to the same bound (or, where the fit is not unique, its residuals); a stop one update away
is accepted only where a stopping test is within reach of the bounds, and its transformation is still held.  The KITTI-shaped
and C2 pairs must be decided at every checked step.  The decided fraction is printed with -s (bounds:
tests/test_icp_fp64_cpu.py)."""
import numpy as np
import pytest
import torch

from oracle import icp_cases as C
from oracle.icp_fp64 import icp_fp64

pytestmark = pytest.mark.gpu

STATS = {"runs": 0, "decided": 0}


def _ops():
    import bufferx_b200 as bx
    return bx.ops


def gpu_icp(c, max_iteration, rel=1e-6):
    ops = _ops()
    dev = torch.device("cuda", torch.cuda.current_device())
    src = torch.from_numpy(np.ascontiguousarray(c["src"], np.float64)).to(dev)
    tgt = torch.from_numpy(np.ascontiguousarray(c["tgt"], np.float64)).to(dev)
    init = torch.from_numpy(np.ascontiguousarray(c["init"], np.float64)).to(dev)
    res, corr = ops.icp(src, tgt, c["r"], init, rel, rel, max_iteration)
    T, fit, rmse, ncorr, iters, conv = ops.decode_icp_result(res.cpu())
    corr = corr[: src.shape[0]].cpu().numpy().astype(np.int64)
    assert ncorr == int((corr >= 0).sum())
    return dict(T=T, fitness=fit, rmse=rmse, corr=corr, iterations=iters, converged=conv, raw=res.cpu().numpy().tobytes())


def run_case(c, ks=None):
    out = icp_fp64(c["src"], c["tgt"], c["r"], init=c["init"], max_iteration=c["max_iteration"])
    n_it = out["iterations"]
    ks = range(n_it + 1) if ks is None else sorted(set(k for k in ks if k <= n_it) | {n_it})
    all_decided, worst = True, 0.0
    for k in ks:
        g = gpu_icp(c, k)
        decided, ratios = C.check_step(g, out, k, c["src"], c["r"], c["hold"])
        STATS["runs"] += 1
        STATS["decided"] += int(decided)
        all_decided &= decided
        worst = max(worst, ratios["rmse"], ratios["T"])
    g = gpu_icp(c, c["max_iteration"])
    if g["iterations"] == n_it:
        assert g["converged"] == out["converged"]
        worst = max(worst, C.check_final(g, out, c["src"], c["tgt"], c["r"], c["hold"]))
    else:
        # a different stop is only allowed where a stopping test is within reach of the bounds, and then by one update,
        # with the final transformation still held
        assert C.stop_marginal(out, max(g["iterations"], n_it), c["src"], c["r"], c["hold"], g), \
            f"stopped after {g['iterations']} updates, the oracle after {n_it}, and no stopping test was marginal"
        worst = max(worst, C.check_final_off_by_one(g, out, c["src"]))
    return out, g, all_decided, worst


@pytest.mark.parametrize("name", C.EDGE)
def test_edge_case(name):
    c = C.case(name)
    out, g, decided, worst = run_case(c)
    print(f"icp {name}: {out['iterations']} updates, decided {decided}, worst ratio {worst:.3g}")
    if c["T_true"] is not None:
        assert np.abs(g["T"] - c["T_true"]).max() < 1e-9 * (1 + np.abs(c["tgt"]).max())
    if name == "none":
        assert g["fitness"] == 0.0 and g["rmse"] == 0.0 and g["iterations"] == 1 and np.array_equal(g["T"], np.eye(4))
    if name == "at_r":
        assert list(gpu_icp(c, 0)["corr"]) == [-1, -1, -1, 3]        # d2 == r*r exactly: no correspondence


@pytest.mark.parametrize("seed", [0, 1])
def test_kitti_call_shape(seed):
    """r = 0.20, init = I, 200 iterations on C3-sized scan pairs pre-aligned by a perturbed ground truth."""
    c = C.kitti_pair(seed)
    out, g, decided, worst = run_case(c, ks=[0, 1, 2, 3, 5, 8, 13, 21])
    print(f"icp kitti seed {seed}: {out['iterations']} updates, fitness {out['fitness']:.4f} rmse {out['rmse']:.4f}, "
          f"decided {decided}, worst ratio {worst:.3g}")
    assert decided, "a KITTI-shaped pair had an undecided step"
    assert g["iterations"] == out["iterations"] and out["fitness"] > 0.9


def test_c2_indoor_pair():
    c = C.c2_pair(0)
    out, g, decided, worst = run_case(c, ks=[0, 1, 2, 4, 8])
    print(f"icp c2: {out['iterations']} updates, decided {decided}, worst ratio {worst:.3g}")
    assert decided, "the C2 pair had an undecided step"
    assert g["iterations"] == out["iterations"]


def test_bit_identical_reruns():
    c = C.kitti_pair(0, n=30000)
    a, b = gpu_icp(c, 200), gpu_icp(c, 200)
    assert a["raw"] == b["raw"] and np.array_equal(a["corr"], b["corr"])


class _O3dCloud:
    def __init__(self, pts):
        self.points = pts


def test_registration_icp_with_open3d_shaped_arguments():
    """The KITTI loader's call with only its import changed."""
    from bufferx_b200 import registration as reg_icp
    c = C.kitti_pair(1, n=40000)
    reg = reg_icp.registration_icp(_O3dCloud(c["src"]), _O3dCloud(c["tgt"]), 0.20, np.eye(4),
                                   reg_icp.TransformationEstimationPointToPoint(),
                                   reg_icp.ICPConvergenceCriteria(max_iteration=200))
    g = gpu_icp(c, 200)
    assert np.array_equal(reg.transformation, g["T"]) and reg.fitness == g["fitness"] and reg.inlier_rmse == g["rmse"]
    cs = np.asarray(reg.correspondence_set)
    assert cs.shape == (int((g["corr"] >= 0).sum()), 2) and (np.diff(cs[:, 0]) > 0).all()
    assert np.array_equal(cs[:, 1], g["corr"][cs[:, 0]])
    # a CUDA tensor source and an array target go through the same coercion
    dev = torch.device("cuda", torch.cuda.current_device())
    reg2 = reg_icp.registration_icp(torch.from_numpy(c["src"]).to(dev), c["tgt"], 0.20,
                                    criteria=reg_icp.ICPConvergenceCriteria(max_iteration=200))
    assert np.array_equal(reg2.transformation, reg.transformation)


def test_decided_fraction():
    """Runs after the cases above (file order): the share of per-step GPU runs whose every decision was out of reach."""
    if STATS["runs"] == 0:
        pytest.skip("no runs recorded (run the whole file)")
    frac = STATS["decided"] / STATS["runs"]
    print(f"icp {STATS['runs']} per-step runs, decided fraction {frac:.3f}")
    assert frac >= 0.5
