"""Edge inputs for point-to-point ICP and the float64 checks the GPU runs are held to, shared by tests/test_icp_*.py (the
bounds are derived in the docstring of tests/test_icp_fp64_cpu.py).  TEST INFRASTRUCTURE ONLY.

``case(name)`` -> dict(src, tgt (float64 [N,3]), r, init (4x4), max_iteration, T_true (or None), hold="T" | "residuals").
``check_step(gpu, step, ...)`` compares one GPU run stopped after k updates with the oracle's step k and returns
(decided, ratios); ``check_final`` holds the final transformation.
"""
import math

import numpy as np

U53 = 2.0 ** -53


def _rot(axis, deg):
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    t = math.radians(deg)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + math.sin(t) * K + (1 - math.cos(t)) * (K @ K)


def _se3(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def apply(T, p):
    return p @ T[:3, :3].T + T[:3, 3]


def _blob(rng, n, spread):
    return rng.uniform(-spread, spread, (n, 3))


def kitti_pair(seed, n=None):
    """The KITTI call shape (synth.kitti_icp_pair): a C3-sized scan pair pre-aligned by a perturbed ground truth, r = 0.20,
    init = I, 200 iterations."""
    from bufferx_b200.synth import kitti_icp_pair
    src, tgt = kitti_icp_pair(seed, n)
    return dict(src=src, tgt=tgt, r=0.20, init=np.eye(4), max_iteration=200, T_true=None, hold="T")


def c2_pair(seed=0):
    """A C2-sized indoor pair pre-aligned the same way, r = 0.1."""
    from bufferx_b200.synth import make_pair
    d = make_pair("C2", seed)
    rng = np.random.default_rng(seed + 99)
    T_gt = np.asarray(d["relt_pose"], np.float64)
    P = _se3(_rot(rng.normal(size=3), 1.0), rng.normal(size=3) * 0.02)
    src = apply(P @ T_gt, d["src_fds_pcd"].astype(np.float64))
    return dict(src=src, tgt=d["tgt_fds_pcd"].astype(np.float64), r=0.1, init=np.eye(4), max_iteration=60, T_true=None, hold="T")


def case(name, seed=0):
    rng = np.random.default_rng(seed + 1000 * len(name))
    base = dict(init=np.eye(4), max_iteration=30, T_true=None, hold="T")
    if name == "exact":
        # noise-free full overlap, a known small rigid motion; target points 0.1 apart, motion beyond the first nearest match
        tgt = _blob(rng, 400, 1.0)
        T = _se3(_rot([1, 2, 3], 4.0), [0.03, -0.02, 0.01])
        return dict(base, src=apply(np.linalg.inv(T), tgt), tgt=tgt, r=0.5, T_true=T, max_iteration=60)
    if name == "init":
        # a non-identity init: the motion is split between init and the ICP updates
        tgt = _blob(rng, 400, 1.0)
        T = _se3(_rot([0, 1, 1], 25.0), [0.4, 0.1, -0.3])
        init = _se3(_rot([0, 1, 1], 22.0), [0.35, 0.12, -0.28])
        return dict(base, src=apply(np.linalg.inv(T), tgt), tgt=tgt, r=0.5, init=init, T_true=T, max_iteration=60)
    if name == "offset":
        # the exact case 1e4 m from the origin
        c = np.array([1e4, -0.6e4, 0.3e4])
        tgt = _blob(rng, 400, 1.0) + c
        T = _se3(_rot([1, 2, 3], 3.0), [0.02, -0.02, 0.01])
        T = _se3(T[:3, :3], T[:3, 3] + c - T[:3, :3] @ c)               # the motion about the cloud's centre
        return dict(base, src=apply(np.linalg.inv(T), tgt), tgt=tgt, r=0.5, T_true=T, max_iteration=60)
    if name == "none":
        # no correspondence at all: identity, fitness 0, rmse 0, one step
        tgt = _blob(rng, 50, 1.0)
        return dict(base, src=_blob(rng, 60, 1.0) + 10.0, tgt=tgt, r=0.5, T_true=np.eye(4))
    if name == "dup":
        # every target point twice (exact ties: the lowest index wins)
        t = _blob(rng, 200, 1.0)
        tgt = np.concatenate([t, t[::-1]])
        T = _se3(_rot([3, 1, 2], 2.0), [0.01, 0.02, -0.01])
        return dict(base, src=apply(np.linalg.inv(T), t), tgt=tgt, r=0.3, T_true=T)
    if name == "at_r":
        # dyadic points whose d2 is exactly r*r = 0.25 (decided in float64: no correspondence under the strict test)
        tgt = np.array([[0.0, 0.0, 0.0], [4.0, 0.0, 0.0], [0.0, 4.0, 0.0], [0.0, 0.0, 4.0]])
        src = tgt + np.array([[0.5, 0.0, 0.0], [0.0, 0.5, 0.0], [0.0, 0.0, -0.5], [0.25, 0.0, 0.0]])
        return dict(base, src=src, tgt=tgt, r=0.5, max_iteration=1)
    if name == "one":
        return dict(base, src=np.array([[0.1, 0.2, 0.3]]), tgt=np.array([[0.15, 0.1, 0.35], [5.0, 5.0, 5.0]]), r=0.5, hold="residuals")
    if name == "two":
        tgt = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [7.0, 7.0, 7.0]])
        src = np.array([[0.05, 0.02, 0.0], [1.02, -0.03, 0.01]])
        return dict(base, src=src, tgt=tgt, r=0.3, hold="residuals")
    if name == "planar":
        # a planar target: rotation about its normal is free, the residuals are held, not R
        tgt = np.c_[rng.uniform(-1, 1, (400, 2)), np.zeros(400)]
        src = apply(_se3(_rot([1, 0, 0], 2.0), [0.0, 0.0, 0.05]), tgt[rng.permutation(400)[:300]] + [0.01, 0.0, 0.0])
        return dict(base, src=src, tgt=tgt, r=0.3, hold="residuals")
    if name == "single":
        # N_src = 1
        return dict(base, src=np.array([[0.3, -0.2, 0.1]]), tgt=_blob(rng, 100, 1.0), r=0.5, hold="residuals")
    if name == "mirror":
        # the best orthogonal map is a reflection (z -> -z of a flat slab): the determinant fix must keep R a rotation
        tgt = np.c_[rng.uniform(-1, 1, (300, 2)), rng.uniform(-0.02, 0.02, 300)]
        src = tgt * [1.0, 1.0, -1.0] + [0, 0, 0.001]
        return dict(base, src=src, tgt=tgt, r=0.2, max_iteration=1, hold="residuals")
    if name == "scaled":
        # target 1 % larger than the source about their centre: the rigid fit keeps R orthonormal
        src = _blob(rng, 300, 1.0)
        return dict(base, src=src, tgt=src * 1.01, r=0.3, max_iteration=5, hold="residuals")
    raise ValueError(name)


EDGE = ("exact", "init", "offset", "none", "dup", "at_r", "one", "two", "planar", "single", "mirror", "scaled")


# --------------------------------------------------------------------------------------------------------------------
# bounds (derivation: tests/test_icp_fp64_cpu.py)
KD = 16.0      # incremental transform: each application moves a coordinate by at most KD u53 (|p| + |t|)
KS = 64.0      # the reductions: sum d2 and the moments, relative KS (n + 16) u53 of their magnitude
KT = 2.0 ** 12  # one Umeyama solve on equal correspondences: |dR|_F <= KT u53 (1 + kappa), kappa = s1 / (s2 + s3)


def _kappa(sv):
    return sv[0] / max(sv[1] + sv[2], 1e-300) if sv[0] > 0 else 0.0


def t_bound(out, k, src):
    """A-priori bound on (|dR|_F, |dt|) between the GPU's and the oracle's transformation after k updates on equal
    correspondences: |dR|_F <= KT u53 sum_{j<=k} (1 + kappa_j), |dt| <= that times (|src centroid| + 1 + |t_k|).  It comes
    from the oracle's own Sigmas, never from the GPU's result, so a drifting GPU transformation cannot widen it."""
    kap = sum(1.0 + _kappa(st["sv"]) for st in out["steps"][1:k + 1])
    bR = KT * U53 * max(kap, 1.0)
    bt = bR * (float(np.linalg.norm(src.mean(0))) + 1.0 + float(np.linalg.norm(out["steps"][k]["T"][:3, 3])))
    return bR, bt


def t_diff(T_gpu, T_or):
    return float(np.linalg.norm(T_gpu[:3, :3] - T_or[:3, :3])), float(np.linalg.norm(T_gpu[:3, 3] - T_or[:3, 3]))


def delta(dR, dt, T_or, src, k):
    """Bound on the distance between the GPU's and the oracle's transformed source points after k updates, for
    transformations that differ by at most (dR, dt)."""
    X = float(np.abs(src).max()) * math.sqrt(3)
    tmax = max(float(np.abs(T_or[:3, 3]).max()), 1.0)
    return dR * X + dt + 2 * (k + 1) * KD * U53 * (X + tmax)


def undecided(step, r, d):
    """Source points whose decision can move when the points move by at most d: |d2 - r^2| or the gap to the second
    neighbour within the possible change of d2, |d d2| <= (2r + d) d (each side) + rounding."""
    D = 2.0 * (2 * r + d) * d + 8 * U53 * r * r
    return int(((step["margin_r"] <= D) | (step["margin_gap"] <= 2 * D)).sum())


def step_delta(gpu, out, k, src, hold):
    """-> (point bound delta_k, ratio of the transformation's error to its bound).  delta_k is built from the measured
    difference of the two transformations (the actual perturbation, so the classification of decisions is sound).  hold 'T':
    that difference must first lie within the a-priori t_bound, so a drifting GPU transformation fails here instead of
    widening the tolerances.  hold 'residuals' (the fit is not unique, so no a-priori bound on T exists): the final residuals
    are held instead (check_final)."""
    T_or = out["steps"][k]["T"]
    dR, dt = t_diff(gpu["T"], T_or)
    if hold != "T":
        return delta(dR, dt, T_or, src, k), 0.0
    bR, bt = t_bound(out, k, src)
    assert dR <= bR and dt <= bt, f"step {k}: T differs by |dR| {dR:.3g} (bound {bR:.3g}), |dt| {dt:.3g} (bound {bt:.3g})"
    return delta(dR, dt, T_or, src, k), max(dR / bR, dt / bt)


def rmse_bound(d, m, nc, n, rmse, r):
    b = d + KS * (n + 16) * U53 * max(rmse, r)
    return b + (r * math.sqrt(2.0 * m / max(nc - m, 1)) if m else 0.0)


def check_step(gpu, out, k, src, r, hold):
    """gpu: dict(T, fitness, rmse, corr, iterations) of a GPU run with max_iteration = k; out: the oracle's run.
    -> (decided, dict of err / bound ratios).  Raises AssertionError when a bound is broken."""
    step = out["steps"][k]
    n = src.shape[0]
    d, rT = step_delta(gpu, out, k, src, hold)
    m = undecided(step, r, d)
    nc = int((step["corr"] >= 0).sum())
    if m == 0:
        assert np.array_equal(gpu["corr"], step["corr"]), f"step {k}: decided correspondences differ"
        assert gpu["fitness"] == step["fitness"], (gpu["fitness"], step["fitness"])
    else:
        diff = int((gpu["corr"] != step["corr"]).sum())
        assert diff <= m, f"step {k}: {diff} correspondences differ, only {m} are undecided"
        assert abs(gpu["fitness"] - step["fitness"]) <= m / n + 1e-15
    b_rmse = rmse_bound(d, m, nc, n, step["rmse"], r)
    ratios = dict(rmse=abs(gpu["rmse"] - step["rmse"]) / b_rmse, T=rT)
    assert ratios["rmse"] <= 1.0, f"step {k}: rmse {gpu['rmse']} vs {step['rmse']} (bound {b_rmse:.3g})"
    return m == 0, ratios


def stop_marginal(out, k, src, r, hold, gpu):
    """True when the stopping test of some step up to k lies within reach of the rmse bound (twice: both rmse values move)
    or an undecided point could move fitness across it -- the only case in which the GPU may stop one update earlier or
    later than the oracle."""
    st = out["steps"]
    n = src.shape[0]
    for j in range(1, min(k, len(st) - 1) + 1):
        d = delta(*t_bound(out, j, src), st[j]["T"], src, j) if hold == "T" else delta(*t_diff(gpu["T"], st[j]["T"]), st[j]["T"], src, j)
        m = max(undecided(st[j], r, d), undecided(st[j - 1], r, d))
        b = 2 * rmse_bound(d, m, int((st[j]["corr"] >= 0).sum()), n, st[j]["rmse"], r)
        if abs(abs(st[j]["fitness"] - st[j - 1]["fitness"]) - 1e-6) <= 2 * m / n or abs(abs(st[j]["rmse"] - st[j - 1]["rmse"]) - 1e-6) <= b:
            return True
    return False


def check_final(gpu, out, src, tgt, r, hold):
    """The final transformation of a run that stopped after as many updates as the oracle's: 'T' -- within t_bound at the
    last step; 'residuals' -- the GPU's own correspondences fit no worse than the oracle's (the fit is not unique: planar
    targets, one or two correspondences)."""
    if hold == "T":
        k = out["iterations"]
        bR, bt = t_bound(out, k, src)
        dR, dt = t_diff(gpu["T"], out["T"])
        assert dR <= bR and dt <= bt, f"T differs: |dR| {dR:.3g} (bound {bR:.3g}), |dt| {dt:.3g} (bound {bt:.3g})"
        return max(dR / bR, dt / bt)
    R = gpu["T"][:3, :3]
    assert np.allclose(R.T @ R, np.eye(3), atol=1e-12) and np.linalg.det(R) > 0
    from oracle.icp_fp64 import xform
    c = gpu["corr"] >= 0
    res = lambda T, cc: float(np.sqrt(np.mean(np.sum((xform(T, src[cc >= 0]) - tgt[cc[cc >= 0]]) ** 2, axis=1)))) if (cc >= 0).any() else 0.0
    e_gpu, e_or = res(gpu["T"], gpu["corr"]), res(out["T"], out["corr"])
    assert int(c.sum()) == int((out["corr"] >= 0).sum())
    assert e_gpu <= e_or + 1e-9 * (1 + r), f"residual {e_gpu} vs oracle {e_or}"
    return 0.0


def check_final_off_by_one(gpu, out, src):
    """A run whose stop was marginal and that stopped one update earlier or later than the oracle: its transformation is
    held against the oracle's final one within t_bound plus the size of the oracle's update at the step where the two
    stops differ (the one update one side applied and the other did not)."""
    k_or, k_g = out["iterations"], gpu["iterations"]
    assert abs(k_g - k_or) == 1, (k_g, k_or)
    st = out["steps"]
    j = max(k_g, k_or) if max(k_g, k_or) < len(st) else k_or
    u = st[j]["update"]
    bR, bt = t_bound(out, k_or, src)
    uR, ut = t_diff(u, np.eye(4))
    dR, dt = t_diff(gpu["T"], out["T"])
    bR2, bt2 = bR + 2 * uR, bt + 2 * (ut + uR * float(np.abs(src).max()) * math.sqrt(3))
    assert dR <= bR2 and dt <= bt2, f"T differs: |dR| {dR:.3g} (bound {bR2:.3g}), |dt| {dt:.3g} (bound {bt2:.3g})"
    return max(dR / bR2, dt / bt2)
