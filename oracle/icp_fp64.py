"""Float64 oracle of point-to-point ICP (csrc/bx_icp.cu, bufferx_b200.registration) -- TEST INFRASTRUCTURE ONLY.

``icp_fp64`` restates Open3D 0.18 ``registration_icp`` with ``TransformationEstimationPointToPoint(with_scaling=False)``
literally, in NumPy float64:
  1. max_correspondence_distance r <= 0 is refused.
  2. pcd = source; if init is not the identity, pcd is transformed by init.  transformation = init.
  3. Evaluation: for each source point the nearest target point with d2 < r*r, d2 = ((dx*dx)+(dy*dy))+(dz*dz) in float64
     (the lowest target index among equal d2); fitness = correspondences / N_src; inlier_rmse = sqrt(sum d2 / correspondences);
     both 0 without a correspondence.
  4. for i < max_iteration: update = umeyama(pcd[c0], target[c1]) (the identity without a correspondence);
     transformation = update @ transformation; pcd = update applied to pcd (incrementally, each coordinate
     ((u0*x + u1*y) + u2*z) + u3); re-evaluate; stop when |d fitness| < relative_fitness and |d rmse| < relative_rmse.
  5. umeyama is Eigen's: centroids, Sigma = (1/n) sum (t - t_mean)(s - s_mean)^T, SVD, S = I with S_33 = -1 when
     det U * det V < 0, R = U S V^T, t = t_mean - R s_mean.
Two rules are assumptions (Open3D leaves them to FLANN): the radius test is strict, and ties go to the lowest target index.
Neighbours come from scipy's cKDTree (the candidates within 2r, 4 per point), their d2 recomputed in the order above.

Every step (0 = the evaluation before the first update) records the correspondences (target index or -1 per source point),
fitness, rmse, the transformation, the update and the singular values of its Sigma, and the margins of its decisions per
source point: ``margin_r`` = |d2_nearest - r*r| (d2_nearest of the nearest target within 2r; 3 r^2 when there is none) and
``margin_gap`` = d2_second - d2_nearest for a point with a correspondence (the gap to the second-nearest target; inf otherwise).

``_mutations`` (test-only) switches the oracle to a wrong variant, so that tests/test_icp_fp64_cpu.py can show that it notices:
"le" (d2 <= r*r), "retransform" (pcd = transformation applied to the source), "right_mul" (transformation @ update),
"no_det_fix", "with_scaling", "fitness_only" (stop on |d fitness| alone), "origin_moments" (Sigma from sums about the origin).
"""
import numpy as np
from scipy.spatial import cKDTree

KNN = 4


def xform(T, p):
    """T [4,4] applied to p [N,3] in the fixed order ((T0*x + T1*y) + T2*z) + T3 per row."""
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    out = np.empty_like(p)
    for r in range(3):
        out[:, r] = (((T[r, 0] * x) + (T[r, 1] * y)) + (T[r, 2] * z)) + T[r, 3]
    return out


def d2_fixed(q, p):
    dx, dy, dz = q[..., 0] - p[..., 0], q[..., 1] - p[..., 1], q[..., 2] - p[..., 2]
    return ((dx * dx) + (dy * dy)) + (dz * dz)


def evaluate(pcd, tgt, tree, r, mutations=()):
    """-> (corr [N] int64 (-1 = none), d2 of the correspondence [N] (0 without), per point |d2_nearest - r*r| [N], per point
    d2_second - d2_nearest [N] (inf without a correspondence))."""
    n = pcd.shape[0]
    k = min(KNN, tgt.shape[0])
    _, idx = tree.query(pcd, k=k, distance_upper_bound=2.0 * r)
    idx = idx.reshape(n, k)
    valid = idx < tgt.shape[0]
    safe = np.where(valid, idx, 0)
    d2 = np.where(valid, d2_fixed(pcd[:, None, :], tgt[safe]), np.inf)
    ids = np.where(valid, idx, np.iinfo(np.int64).max)
    order = np.lexsort((ids, d2), axis=-1)                 # each row by d2, then by index (the tie rule)
    d2s = np.take_along_axis(d2, order, 1)
    ids = np.take_along_axis(ids, order, 1)
    r2 = r * r
    d1 = d2s[:, 0]
    hit = (d1 <= r2) if "le" in mutations else (d1 < r2)
    corr = np.where(hit, ids[:, 0], -1)
    mr = np.where(np.isfinite(d1), np.abs(d1 - r2), 3.0 * r2)
    with np.errstate(invalid="ignore"):
        mg = np.where(hit, (d2s[:, 1] - d1) if k > 1 else np.inf, np.inf)
    return corr, np.where(hit, d1, 0.0), mr, mg


def umeyama(s, t, mutations=()):
    """Eigen::umeyama(s^T, t^T, with_scaling) for [n,3] float64 point sets -> (4x4 (the identity when n == 0), singular values
    of Sigma)."""
    T = np.eye(4)
    n = s.shape[0]
    if n == 0:
        return T, np.zeros(3)
    ms, mt = s.mean(0), t.mean(0)
    sd, td = s - ms, t - mt
    if "origin_moments" in mutations:
        sigma = (t.T @ s) / n - np.outer(mt, ms)
    else:
        sigma = (td.T @ sd) / n
    U, D, Vt = np.linalg.svd(sigma)
    S = np.ones(3)
    if "no_det_fix" not in mutations and np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2] = -1.0
    R = U @ np.diag(S) @ Vt
    if "with_scaling" in mutations:
        R = R * (float((D * S).sum()) / float((sd * sd).sum() / n))
    T[:3, :3] = R
    T[:3, 3] = mt - R @ ms
    return T, D


def icp_fp64(source, target, max_correspondence_distance, init=None, relative_fitness=1e-6, relative_rmse=1e-6,
             max_iteration=30, _mutations=()):
    """-> dict(T, fitness, rmse, corr, iterations (updates applied), converged, pcd (final), steps=[dict(corr, fitness, rmse,
    T, update, sv (singular values of the update's Sigma), margin_r, margin_gap)])."""
    r = float(max_correspondence_distance)
    if not r > 0.0:
        raise ValueError(f"max_correspondence_distance must be positive, got {r}")
    src = np.asarray(source, np.float64).reshape(-1, 3)
    tgt = np.asarray(target, np.float64).reshape(-1, 3)
    if src.shape[0] == 0 or tgt.shape[0] == 0:
        raise ValueError("empty cloud")
    T = np.eye(4) if init is None else np.array(init, np.float64).reshape(4, 4)
    tree = cKDTree(tgt)
    pcd = src.copy() if np.array_equal(T, np.eye(4)) else xform(T, src)
    corr, d2, mr, mg = evaluate(pcd, tgt, tree, r, _mutations)

    def result(corr, d2):
        n = int((corr >= 0).sum())
        return (n / src.shape[0], float(np.sqrt(d2.sum() / n))) if n else (0.0, 0.0)

    fit, rmse = result(corr, d2)
    steps = [dict(corr=corr, fitness=fit, rmse=rmse, T=T.copy(), update=np.eye(4), sv=np.zeros(3), margin_r=mr, margin_gap=mg)]
    converged = False
    for _ in range(int(max_iteration)):
        c = corr >= 0
        upd, sv = umeyama(pcd[c], tgt[corr[c]], _mutations)
        T = T @ upd if "right_mul" in _mutations else upd @ T
        pcd = xform(T, src) if "retransform" in _mutations else xform(upd, pcd)
        corr, d2, mr, mg = evaluate(pcd, tgt, tree, r, _mutations)
        pf, pr = fit, rmse
        fit, rmse = result(corr, d2)
        steps.append(dict(corr=corr, fitness=fit, rmse=rmse, T=T.copy(), update=upd, sv=sv, margin_r=mr, margin_gap=mg))
        if abs(pf - fit) < relative_fitness and ("fitness_only" in _mutations or abs(pr - rmse) < relative_rmse):
            converged = True
            break
    return dict(T=T, fitness=fit, rmse=rmse, corr=corr, iterations=len(steps) - 1, converged=converged, pcd=pcd, steps=steps)
