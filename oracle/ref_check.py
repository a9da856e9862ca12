"""Pin the oracle against the REFERENCE's own Python, and write the golden fixtures.

    python oracle/ref_check.py            # needs /root/reference (build container only)

TEST INFRASTRUCTURE (not product).  What it does:
  1. puts /root/reference on sys.path and imports the reference's ``models.BUFFERX.BufferX``,
     ``config``-style cfg, ``utils.common`` ... UNMODIFIED;
  2. supplies the third-party leaf modules that are absent from this image and from
     /root/reference (pointnet2_ops, knn_cuda, torch_batch_svd, kornia, open3d, easydict,
     matplotlib) as thin stubs whose leaf ops are the restatements in oracle/oracle.py
     (pointnet2 FPS / ball query / gather / group, kNN, Open3D RANSAC) or torch built-ins
     (SVD, Rodrigues); ``Tensor.cuda()`` becomes a no-op so the reference runs on CPU;
  3. runs the reference ``BufferX.forward`` (inference branch, models/BUFFERX.py:257-467) on synthetic
     pairs (default: the full C2 configuration -- 2x20000 points, 1500 key-points, 3 scales, 50000 RANSAC
     iterations -- seeds 0, 1, 2, with the FITTED CostNet so that the run ends in a non-trivial consensus
     set, RANSAC and refinement) with the same weights / permutation seed, captures every stage through
     forward hooks, and compares with ``oracle.register_pair`` three times:
       oracle_free        the oracle on its own (literal Rodrigues, own covariance sum + Jacobi);
       oracle_zlocked     the oracle with the reference run's LRF z axes imposed: the covariance sum is a
                          BLAS call in the reference (summation order not in its source), everything
                          downstream of it must agree exactly -> identical match lists, consensus set,
                          RANSAC result and pose;
       oracle_stable_form the round-1 well-conditioned Rodrigues form (BX_LRF=stable), for the sensitivity
                          report (fraction of descriptors / matches that change);
     this pins all the glue (indexing, masks, layouts, concatenation order, radius bisection, conv stacks,
     cost volume, hypothesis build, consensus, refinement) that IS in /root/reference;
  4. writes tests/golden/<workload>_seed<k>.npz (oracle outputs = what the CUDA path must reproduce),
     <...>_reference.npz (what the reference produced, including its z axes, so that the z-locked
     comparison is replayed by tests/test_oracle_cpu.py without /root/reference) and <...>_report.json.
The script itself is committed so the fixtures can be regenerated:
    python oracle/ref_check.py --workload C2 --seeds 0 1 2      # ~4 min per seed on 8 cores
    python oracle/ref_check.py --workload C1 --seeds 0 --untrained
    python oracle/ref_check.py --workload C3 --seeds 0 1        # the reduced routes of ROUTES below, likewise C5 --seeds 0,
    python oracle/ref_check.py --workload C3L --seeds 0         # C3LT / C3LE --seeds 0, C2E / C2N --seeds 0
"""
from __future__ import annotations

import hashlib
import json
import os
import sys
import time
import types
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = "/root/reference"
sys.path[:] = [q for q in sys.path if os.path.abspath(q or ".") != HERE]
sys.path.insert(0, ROOT)

import bufferx_b200 as bx  # noqa: E402
from bufferx_b200.se3 import compute_rre, compute_rte  # noqa: E402
from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg  # noqa: E402
from oracle import oracle as O  # noqa: E402


# --------------------------------------------------------------------------------------------- #
# stubs for the third-party modules the reference imports
# --------------------------------------------------------------------------------------------- #
def _mod(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


class _RansacLog:
    calls = []


class _FpsLog:
    calls = []


def install_stubs(ransac_seed=0):
    # easydict
    from bufferx_b200.easydict import EasyDict
    _mod("easydict", EasyDict=EasyDict)

    # pointnet2_ops.pointnet2_utils
    def furthest_point_sample(xyz, npoint):
        out = torch.stack([torch.from_numpy(O.fps(x.numpy(), npoint)) for x in xyz]).int()
        _FpsLog.calls.append(out[0].numpy().copy())
        return out

    def gather_operation(features, idx):
        return torch.gather(features, 2, idx.long()[:, None, :].expand(-1, features.shape[1], -1))

    def ball_query(radius, nsample, xyz, new_xyz):
        out = [torch.from_numpy(O.ball_query(x.numpy(), q.numpy(), float(radius), nsample)[0]) for x, q in zip(xyz, new_xyz)]
        return torch.stack(out).int()

    def grouping_operation(features, idx):
        B, C, N = features.shape
        _, M, S = idx.shape
        flat = idx.long().reshape(B, 1, M * S).expand(-1, C, -1)
        return torch.gather(features, 2, flat).reshape(B, C, M, S)

    p2 = _mod("pointnet2_ops")
    p2.pointnet2_utils = _mod("pointnet2_ops.pointnet2_utils", furthest_point_sample=furthest_point_sample,
                              gather_operation=gather_operation, ball_query=ball_query,
                              grouping_operation=grouping_operation)

    # knn_cuda
    class KNN:
        def __init__(self, k=1, transpose_mode=True):
            assert k == 1 and transpose_mode

        def __call__(self, ref, query):
            _, _, snn, _ = O.mutual_nn(query[0].numpy(), ref[0].numpy())
            idx = torch.from_numpy(snn.astype(np.int64))[None, :, None]
            d = torch.norm(query[0] - ref[0][idx[0, :, 0]], dim=-1)[None, :, None]
            return d, idx

    _mod("knn_cuda", KNN=KNN)

    # torch_batch_svd
    _mod("torch_batch_svd", svd=lambda a: torch.svd(a))

    # kornia.geometry.conversions.axis_angle_to_rotation_matrix (kornia >= 0.7 formulae)
    def axis_angle_to_rotation_matrix(axis_angle):
        def _normal(aa, theta2, eps=1e-6):
            theta = torch.sqrt(theta2)
            wxyz = aa / (theta + eps)
            wx, wy, wz = torch.chunk(wxyz, 3, dim=1)
            c, s = torch.cos(theta), torch.sin(theta)
            k1 = 1.0
            r = [c + wx * wx * (k1 - c), wx * wy * (k1 - c) - wz * s, wy * s + wx * wz * (k1 - c),
                 wz * s + wx * wy * (k1 - c), c + wy * wy * (k1 - c), -wx * s + wy * wz * (k1 - c),
                 -wy * s + wx * wz * (k1 - c), wx * s + wy * wz * (k1 - c), c + wz * wz * (k1 - c)]
            return torch.cat(r, dim=1).view(-1, 3, 3)

        def _taylor(aa):
            rx, ry, rz = torch.chunk(aa, 3, dim=1)
            one = torch.ones_like(rx)
            return torch.cat([one, -rz, ry, rz, one, -rx, -ry, rx, one], dim=1).view(-1, 3, 3)

        aa = torch.unsqueeze(axis_angle, dim=1)
        theta2 = torch.matmul(aa, aa.transpose(1, 2)).squeeze(1)
        Rn, Rt = _normal(axis_angle, theta2), _taylor(axis_angle)
        mask = (theta2 > 1e-6).view(-1, 1, 1).type_as(theta2)
        out = torch.eye(3).to(axis_angle).view(1, 3, 3).repeat(axis_angle.shape[0], 1, 1)
        out[..., :3, :3] = mask * Rn + (1 - mask) * Rt
        return out

    k = _mod("kornia")
    k.geometry = _mod("kornia.geometry")
    k.geometry.conversions = _mod("kornia.geometry.conversions", axis_angle_to_rotation_matrix=axis_angle_to_rotation_matrix)

    # matplotlib (visualisation only)
    mpl = _mod("matplotlib")
    mpl.colors = _mod("matplotlib.colors")
    mpl.cm = _mod("matplotlib.cm")
    mpl.pyplot = _mod("matplotlib.pyplot")

    # open3d: just enough for utils/common.py::make_open3d_point_cloud and pose_estimator.py:84-117
    class _Vec(np.ndarray):
        pass

    def _vec(a):
        return np.asarray(a)

    class PointCloud:
        def __init__(self):
            self.points = None
            self.colors = None

    class _Result:
        def __init__(self, T, cs):
            self.transformation, self.correspondence_set = T, cs

    class _Crit:
        def __init__(self, max_iteration=100000, confidence=0.999):
            self.max_iteration, self.confidence = max_iteration, confidence

    class _Edge:
        def __init__(self, th):
            self.th = th

    class _Dist:
        def __init__(self, th):
            self.th = th

    def ransac_corr(pcd0, pcd1, corr, max_d, estimation, ransac_n, checkers, criteria):
        corr = np.asarray(corr)
        assert ransac_n == 3 and (corr[:, 0] == corr[:, 1]).all()
        r = O.ransac(np.asarray(pcd0.points, dtype=np.float32), np.asarray(pcd1.points, dtype=np.float32), corr[:, 0],
                     max_d, checkers[0].th, criteria.confidence, criteria.max_iteration, ransac_seed)
        _RansacLog.calls.append(dict(inlier_ind=corr[:, 0].copy(), **r))
        return _Result(r["T"], [0] * r["num_inliers"])

    o3d = _mod("open3d")
    o3d.geometry = _mod("open3d.geometry", PointCloud=PointCloud)
    o3d.utility = _mod("open3d.utility", Vector3dVector=_vec, Vector2iVector=_vec)
    reg = _mod("open3d.pipelines.registration", registration_ransac_based_on_correspondence=ransac_corr,
               TransformationEstimationPointToPoint=lambda s=False: ("p2p", s),
               CorrespondenceCheckerBasedOnEdgeLength=_Edge, CorrespondenceCheckerBasedOnDistance=_Dist,
               RANSACConvergenceCriteria=_Crit)
    o3d.pipelines = _mod("open3d.pipelines", registration=reg)

    torch.Tensor.cuda = lambda self, *a, **k: self  # the reference hard-codes .cuda() (patch_embedder.py:158)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


def _savez(path, **arrays):
    """np.savez_compressed with a fixed member timestamp, so that a rerun writes the same bytes."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k, v in arrays.items():
            zi = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            zi.compress_type = zipfile.ZIP_DEFLATED
            with z.open(zi, "w", force_zip64=True) as f:
                np.lib.format.write_array(f, np.asanyarray(v), allow_pickle=False)


# The routes pinned beside C2.  A full-size C3 reference forward (2048 key-points, 50000 iterations) ran for more than two
# minutes without finishing on 8 cores, so the outdoor routes pin a reduced variant: 300 key-points, 600 radius key-points,
# 5000 RANSAC iterations, everything else (cloud sizes, the 200000-point cut, thresholds, alignment, early-exit rule) as
# configured.  The early-exit routes on C2 keep the full C2 configuration: with 300 key-points scale 0 finds no inlier.
#   geom: synthetic geometry; sizes: (n_src, n_tgt) or None; exit: "at" -> early_exit_min_inliers = the scale-0 RANSAC
#   count (the pair exits, on the >= boundary), "above" -> that count + 1 (it does not).
ROUTES = {
    "C3": dict(geom="C3", sizes=None, exit=None),                   # KITTI: aligned, confidence 1.0, no refinement
    "C5": dict(geom="C5", sizes=None, exit=None),                   # TIERS_hetero, 60000 vs 30000 points
    "C3L": dict(geom="C3", sizes=(260000, 230000), exit=None),      # both above 200000 points, the source larger
    "C3LT": dict(geom="C3", sizes=(240000, 240000), exit=None),     # equal sizes: the target is sub-sampled
    "C3LE": dict(geom="C3", sizes=(260000, 230000), exit="at"),     # above 200000 points, exits after one draw
    "C2E": dict(geom="C2", sizes=None, exit="at"),                  # early exit at scale 0
    "C2N": dict(geom="C2", sizes=None, exit="above"),               # early exit on, the pair does not exit
}


def route_cfg(name):
    """The cfg of a ROUTES workload (early_exit_min_inliers left at the dataset's value; ``main`` sets it)."""
    rt = ROUTES[name]
    cfg = workload_cfg(rt["geom"])
    if rt["geom"] != "C2":
        cfg.patch.num_fps, cfg.patch.num_points_radius_estimate, cfg.match.iter_n = 300, 600, 5000
    cfg.match.enable_early_exit = rt["exit"] is not None
    return cfg


def route_pair(name, seed):
    rt = ROUTES[name]
    ns, nt = rt["sizes"] or (None, None)
    return make_pair(rt["geom"], seed, n_src=ns, n_tgt=nt)


class RandintLog:
    """Records every ``torch.randint`` call made inside the block: count, sha of each result, and the sha of torch's CPU
    generator state on exit (the reference's only use of that generator is its radius sub-sample)."""

    def __enter__(self):
        self.shas, self._orig = [], torch.randint

        def rec(*a, **kw):
            t = self._orig(*a, **kw)
            self.shas.append(sha(t.cpu().numpy()))
            return t

        torch.randint = rec
        return self

    def __exit__(self, *exc):
        torch.randint = self._orig
        self.state_sha = sha(torch.get_rng_state().numpy())
        return False


def _workload(name):
    """C1/C2/... as in bufferx_b200.synth; "C1S3" = the C1 geometry with the full three-scale configuration; ROUTES
    names as above."""
    if name == "C1S3":
        cfg = workload_cfg("C1")
        cfg.patch.num_scales = 3
        cfg.patch.search_radius_thresholds = [5, 2, 0.5]
        return cfg, "C1"
    if name in ROUTES:
        return route_cfg(name), ROUTES[name]["geom"]
    return workload_cfg(name), name


def _rel_desc_err(a, b):
    den = b.abs().max(dim=1).values
    return (a - b).abs().max(dim=1).values / torch.where(den > 0, den, torch.ones_like(den))


def _compare(tag, rep, cfg, cap, mm, rlog, ref_out, ora_out):
    """reference run vs one oracle run -> entries of the report under ``tag``."""
    pose_r, ninl_r, nmut_r, nind_r, su_r = ref_out
    pose_o, ninl_o, nmut_o, nind_o, su_o, aux = ora_out
    S = min(su_r, su_o)
    r = {"scales_used": (int(su_r), int(su_o))}
    all_equal = su_r == su_o
    for i in range(S):
        sc = aux["scales"][i]
        for side, j in (("src", 2 * i), ("tgt", 2 * i + 1)):
            rd, od = cap["desc"][j], sc[side]
            dd = _rel_desc_err(rd["desc"], od["desc"])
            r[f"s{i}_{side}_desc_frac_within_1e-4"] = float((dd < 1e-4).float().mean())
            r[f"s{i}_{side}_desc_max_rel"] = float(dd.max())
            r[f"s{i}_{side}_R_maxabs"] = float((rd["R"] - od["R"]).abs().max())
            r[f"s{i}_{side}_patches_maxabs"] = float((rd["patches"] - torch.from_numpy(od["delta"])).abs().max())
        rs, rt = mm[i]
        eq = bool(rs.numel() == len(sc["s_mids"]) and (rs.numpy() == sc["s_mids"]).all() and (rt.numpy() == sc["t_mids"]).all())
        r[f"s{i}_M_ref"], r[f"s{i}_M_oracle"], r[f"s{i}_mids_equal"] = int(rs.numel()), int(len(sc["s_mids"])), eq
        a = set(zip(rs.numpy().tolist(), rt.numpy().tolist()))
        b = set(zip(sc["s_mids"].tolist(), sc["t_mids"].tolist()))
        r[f"s{i}_mids_common"] = len(a & b)
        all_equal &= eq
        if eq:
            r[f"s{i}_ind_maxabs"] = float(np.abs(cap["pose"][i].numpy() - sc["ind"]).max())
    rc = rlog[-1] if rlog else None
    if rc is not None:
        last = aux["scales"][su_o - 1]
        r["inlier_ind_equal"] = bool(len(rc["inlier_ind"]) == len(last["inlier_ind"]) and (rc["inlier_ind"] == last["inlier_ind"]).all())
        r["inlier_ind_ref_oracle_common"] = [int(len(rc["inlier_ind"])), int(len(last["inlier_ind"])),
                                             int(len(np.intersect1d(rc["inlier_ind"], last["inlier_ind"])))]
    oc = aux["ransac_calls"]
    r["ransac_calls"] = (len(rlog), len(oc))
    r["ransac_calls_equal"] = bool(len(rlog) == len(oc) and all(
        np.array_equal(a["inlier_ind"], b["inlier_ind"]) and a["num_inliers"] == b["num_inliers"]
        and np.abs(np.asarray(a["T"]) - b["T"]).max() <= 1e-12 for a, b in zip(rlog, oc)))
    r["des_r_equal"] = bool(list(cap["des_r"]) == list(aux["des_r"]))
    r["all_mids_equal"] = all_equal
    r["num_inliers"] = (int(ninl_r), int(ninl_o))
    r["num_mutual"] = (int(nmut_r), int(nmut_o))
    r["num_inlier_ind"] = (int(nind_r), int(nind_o))
    P_r, P_o = np.asarray(pose_r, dtype=np.float64), np.asarray(pose_o, dtype=np.float64)
    r["pose_maxabs"] = float(np.abs(P_r - P_o).max())
    r["pose_rre_deg"], r["pose_rte_m"] = float(compute_rre(P_o, P_r)), float(compute_rte(P_o, P_r))
    r["pose_is_identity"] = bool(np.abs(P_r - np.eye(4)).max() < 1e-9)
    rep[tag] = r
    return r


def main(workload="C2", seed=0, ransac_seed=0, trained=True, stride=8):
    _RansacLog.calls.clear()
    install_stubs(ransac_seed)
    if REF not in sys.path:
        sys.path.insert(0, REF)
    for m in [k for k in sys.modules if k == "models" or k.startswith("models.") or k == "utils" or k.startswith("utils.")]:
        del sys.modules[m]
    import models.BUFFERX as RB  # the reference's module
    import utils.common as RC     # the reference's utils/common.py

    cfg, geom = _workload(workload)
    ours = init_synthetic_weights(bx.BufferX(cfg), trained_pose=trained)
    sd = {k: v.detach().clone() for k, v in ours.state_dict().items()}
    ref = RB.BufferX(cfg)
    missing = ref.load_state_dict(sd, strict=True)          # pins the state_dict key/shape contract
    ref.eval()
    print("reference state_dict keys == ours:", list(ref.state_dict().keys()) == list(sd.keys()), missing)

    data = route_pair(workload, seed) if workload in ROUTES else make_pair(geom, seed)
    n_s, n_t = data["src_fds_pcd"].shape[0], data["tgt_fds_pcd"].shape[0]
    tdata = {k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in data.items()}
    perms = O.draw_perms(cfg, n_s, n_t, seed)
    S = cfg.patch.num_scales
    exit_mode = ROUTES[workload]["exit"] if workload in ROUTES else None
    if exit_mode is not None:
        # the early-exit threshold sits on the scale-0 RANSAC count, so that the >= of the exit test is what decides
        cfg.match.early_exit_min_inliers = 0
        with torch.random.fork_rng():
            n0 = O.register_pair(sd, cfg, data, perms, ransac_seed)[1]
        cfg.match.early_exit_min_inliers = n0 if exit_mode == "at" else n0 + 1

    cap = dict(desc=[], pose=[], z=[], des_r=[], radius_clouds=[])
    orig_dare = RB.density_aware_radius_estimation
    RB.density_aware_radius_estimation = lambda *a, **k: (lambda r: (cap["des_r"].extend(r), r)[1])(orig_dare(*a, **k))
    # which key-points and which (sub-sampled) points each radius estimation measured: the sha of both
    orig_cdist = RB.squared_cdist
    RB.squared_cdist = lambda x, y: (cap["radius_clouds"].append(sha(x.numpy()) + sha(y.numpy())), orig_cdist(x, y))[1]
    _FpsLog.calls.clear()
    ref.Desc.register_forward_hook(lambda m, i, o: cap["desc"].append({k: (v.detach().clone() if torch.is_tensor(v) else v) for k, v in o.items()}))
    ref.Pose.register_forward_hook(lambda m, i, o: cap["pose"].append(o.detach().clone().reshape(-1)))
    mm = []
    orig_mm = ref.mutual_matching
    ref.mutual_matching = lambda a, b: (lambda r: (mm.append(r), r)[1])(orig_mm(a, b))
    # the z axes the reference hands to its Rodrigues formula (utils/common.py:501: argument `a`)
    orig_rods = RC.RodsRotatFormula
    RC.RodsRotatFormula = lambda a, b: (cap["z"].append(a.detach().clone().numpy()), orig_rods(a, b))[1]

    np.random.seed(seed)                                    # the reference draws its permutations here
    torch.manual_seed(seed)                                 # ... and its radius sub-samples here
    t0 = time.perf_counter()
    with torch.no_grad(), RandintLog() as draws_r:
        pose_r, times, ninl_r, nmut_r, nind_r, su_r = ref(tdata)
    t_ref = time.perf_counter() - t0
    RC.RodsRotatFormula = orig_rods
    RB.density_aware_radius_estimation = orig_dare
    RB.squared_cdist = orig_cdist
    ref_out = (pose_r, ninl_r, nmut_r, nind_r, su_r)
    rlog = list(_RansacLog.calls)

    rep = dict(workload=workload, seed=seed, ransac_seed=ransac_seed, trained_pose=bool(trained),
               reference_forward_seconds=round(t_ref, 1), n_src=int(n_s), n_tgt=int(n_t),
               early_exit_min_inliers=cfg.match.get("early_exit_min_inliers", 15) if exit_mode else None,
               reference_draws=dict(count=len(draws_r.shas), shas=draws_r.shas, state=draws_r.state_sha))

    def oracle_run(tag, **kw):
        torch.manual_seed(seed)
        with RandintLog() as dr:
            out = O.register_pair(sd, cfg, data, perms, ransac_seed, keep=True, **kw)
        _compare(tag, rep, cfg, cap, mm, rlog, ref_out, out)
        rep[tag]["draws_equal"] = bool(dr.shas == draws_r.shas and dr.state_sha == draws_r.state_sha)
        return out

    # (1) the oracle on its own: covariance sum / eigen-solver are its own (the reference's are BLAS / LAPACK calls whose
    #     summation order is not part of its source), everything else literal
    os.environ.pop("BX_LRF", None)
    free = oracle_run("oracle_free")
    # (2) the same with the reference run's own z axes imposed: everything downstream must now agree exactly
    #     (none on the aligned route: it builds no LRF)
    z_axes = None
    if cap["z"]:
        ran = len(cap["z"]) // 2
        z_axes = [(cap["z"][2 * i], cap["z"][2 * i + 1]) for i in range(ran)] + [(None, None)] * (S - ran)
        locked = oracle_run("oracle_zlocked", z_axes=z_axes)
        ang = []
        for i in range(min(ran, free[4])):
            for j, side in ((0, "src"), (1, "tgt")):
                dots = np.clip(np.sum(z_axes[i][j].astype(np.float64) * free[5]["scales"][i][side]["z"].astype(np.float64), axis=1), -1, 1)
                ang.append(np.degrees(np.arccos(dots)))
        ang = np.concatenate(ang)
        rep["z_axis_angle_deg_free_vs_reference"] = dict(median=float(np.median(ang)), p99=float(np.percentile(ang, 99)), max=float(ang.max()),
                                                         sign_flips=int((ang > 90).sum()))
    # (3) sensitivity: the well-conditioned Rodrigues form (round 1's oracle) instead of the literal one (LRF routes only)
    if cap["z"]:
        os.environ["BX_LRF"] = "stable"
        stable = oracle_run("oracle_stable_form")
        os.environ.pop("BX_LRF", None)
        chg_d, chg_m, tot_m = [], 0, 0
        for i in range(min(free[4], stable[4])):
            for side in ("src", "tgt"):
                chg_d.append(_rel_desc_err(stable[5]["scales"][i][side]["desc"], free[5]["scales"][i][side]["desc"]).numpy())
            a = set(zip(free[5]["scales"][i]["s_mids"].tolist(), free[5]["scales"][i]["t_mids"].tolist()))
            b = set(zip(stable[5]["scales"][i]["s_mids"].tolist(), stable[5]["scales"][i]["t_mids"].tolist()))
            chg_m += len(a ^ b)
            tot_m += len(a)
        chg_d = np.concatenate(chg_d)
        rep["literal_vs_stable"] = {"desc_frac_changed_over_1e-4": float((chg_d >= 1e-4).mean()), "desc_frac_changed_at_all": float((chg_d > 0).mean()),
                                    "matches_changed": int(chg_m), "matches_total": int(tot_m)}
    print(json.dumps(rep, indent=1))

    # --- golden fixtures (small: match lists, soft arg-max bins, consensus set, poses, a strided descriptor sample) ---
    pose_o, ninl_o, nmut_o, nind_o, su_o, aux = free
    tag = f"{workload.lower()}_seed{seed}"
    gold_dir = os.path.join(ROOT, "tests", "golden")
    os.makedirs(gold_dir, exist_ok=True)
    if workload not in ROUTES:      # the oracle's own outputs (the route workloads hold the CUDA path to the reference's)
        gold = dict(workload=workload, seed=seed, ransac_seed=ransac_seed, trained_pose=bool(trained), stride=stride,
                    s_fps=aux["s_fps"], t_fps=aux["t_fps"], des_r=np.array(aux["des_r"], dtype=np.float64),
                    pose=np.asarray(pose_o, dtype=np.float64), init_pose=np.asarray(aux["init_pose"], dtype=np.float64),
                    counts=np.array([ninl_o, nmut_o, nind_o, su_o], dtype=np.int64))
        for i in range(S):
            sc = aux["scales"][i]
            for side in ("src", "tgt"):
                d = sc[side]
                gold[f"s{i}_{side}_idx_sha"] = np.frombuffer(sha(d["idx"]).encode(), dtype=np.uint8)
                gold[f"s{i}_{side}_vidx_sha"] = np.frombuffer(sha(d["vidx"]).encode(), dtype=np.uint8)
                gold[f"s{i}_{side}_idx_head"] = d["idx"][:8].copy()
                gold[f"s{i}_{side}_desc"] = d["desc"].numpy()[::stride]
                gold[f"s{i}_{side}_R"] = d["R"].numpy()[::stride]
            gold[f"s{i}_s_mids"], gold[f"s{i}_t_mids"] = sc["s_mids"].astype(np.int32), sc["t_mids"].astype(np.int32)
            gold[f"s{i}_ind"] = sc["ind"]
            gold[f"s{i}_inlier_ind"] = sc["inlier_ind"].astype(np.int32)
        np.savez_compressed(os.path.join(gold_dir, f"{tag}.npz"), **gold)
    # what the REFERENCE's own forward produced (+ its z axes, to replay the z-locked comparison without /root/reference)
    refd = dict(pose=np.asarray(pose_r, dtype=np.float64), counts=np.array([ninl_r, nmut_r, nind_r, su_r], dtype=np.int64), stride=stride)
    if rlog:
        refd["inlier_ind"] = rlog[-1]["inlier_ind"].astype(np.int32)
        refd["ransac_T"] = np.asarray(rlog[-1]["T"], dtype=np.float64)
    for i in range(su_r):
        refd[f"s{i}_src_desc"] = cap["desc"][2 * i]["desc"].numpy()[::stride]
        refd[f"s{i}_tgt_desc"] = cap["desc"][2 * i + 1]["desc"].numpy()[::stride]
        refd[f"s{i}_s_mids"], refd[f"s{i}_t_mids"] = mm[i][0].numpy().astype(np.int32), mm[i][1].numpy().astype(np.int32)
        refd[f"s{i}_ind"] = cap["pose"][i].numpy()
        if z_axes is not None:
            refd[f"s{i}_src_z"], refd[f"s{i}_tgt_z"] = z_axes[i]
    if workload in ROUTES:
        # every RANSAC call, the per-scale radii, the Kr-point FPS of both clouds, the torch generator's draws
        refd.update(n_src=n_s, n_tgt=n_t, seed=seed, early_exit_min_inliers=cfg.match.get("early_exit_min_inliers", 15),
                    s_fps=_FpsLog.calls[0].astype(np.int32), t_fps=_FpsLog.calls[1].astype(np.int32),
                    des_r=np.array(cap["des_r"], dtype=np.float64), n_ransac=len(rlog),
                    n_draws=len(draws_r.shas), rng_state_sha=np.frombuffer(draws_r.state_sha.encode(), dtype=np.uint8))
        for k, c in enumerate(rlog):
            refd[f"ransac{k}_inlier_ind"] = c["inlier_ind"].astype(np.int32)
            refd[f"ransac{k}_T"] = np.asarray(c["T"], dtype=np.float64)
            refd[f"ransac{k}_num_inliers"] = int(c["num_inliers"])
        for k, h in enumerate(draws_r.shas):
            refd[f"draw{k}_sha"] = np.frombuffer(h.encode(), dtype=np.uint8)
        for k, h in enumerate(cap["radius_clouds"]):
            refd[f"radius{k}_cloud_sha"] = np.frombuffer(h.encode(), dtype=np.uint8)
    _savez(os.path.join(gold_dir, f"{tag}_reference.npz"), **refd)
    with open(os.path.join(ROOT, "tests", "golden", f"{tag}_report.json"), "w") as f:
        json.dump(rep, f, indent=1)
    return rep


if __name__ == "__main__":
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="C2", help="C1 | C1S3 | C2, or a reduced route: " + " | ".join(ROUTES))
    ap.add_argument("--seeds", type=int, nargs="+", default=[0, 1, 2])
    ap.add_argument("--untrained", action="store_true", help="random CostNet (round 1's vacuous pin) instead of the fitted one")
    ap.add_argument("--stride", type=int, default=None, help="key-point stride of the descriptor sample kept in the fixture (default 8; 1 for C1)")
    a = ap.parse_args()
    for sd_ in a.seeds:
        main(a.workload, sd_, 0, trained=not a.untrained, stride=a.stride or (1 if a.workload == "C1" else 8))
