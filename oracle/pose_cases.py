"""Edge inputs for mutual matching, consensus, RANSAC and refinement (a10, a13-a15) and the float64 checks they are held
to, shared by tests/test_pose_fp64_*.py (the derivation of every bound is in the docstring of tests/test_pose_fp64_cpu.py).

TEST INFRASTRUCTURE ONLY.  ``corr_set(kind, n)`` builds fp32 correspondences (ss, tt): generic, planar, mirrored (the
best orthogonal map has det -1), near-collinear, exactly collinear, coincident, 180-degree rotations (quaternion w = 0),
identity, spreads from 1e-3 m to 80 m and offsets 0, 80 m, 1e3 and 1e4 m.  ``desc_set(Ka, Kb)`` builds descriptors:
random unit rows, exact duplicates, all-zero rows and rows one ulp apart.  The ``check_*`` functions assert the bounds
and return the largest ratio (err / bound) of each check and the number of decisions left to rounding."""
import numpy as np

from . import oracle as O

F32 = np.float32
U = 2.0 ** -24                 # fp32 unit roundoff
U53 = O.U53                    # fp64 unit roundoff

KN = 4.0                       # matching distances: |fl32(d) - d64| <= KN (C + 3) u d64
KC = 8.0                       # consensus: fp32 transform, difference, norm and threshold
KF = 32.0                      # fp64 fits: |dH| <= KF u53 sum |a - ca| |b - cb|
KR = 4.0                       # fp32 output rounding of a refined pose
KD = 8.0                       # refinement distances in fp32

DIST_TH = (0.10, 0.20, 0.30)
SIMILAR_TH = (0.8, 0.9)
INLIER_TH = (1 / 3, 1.5, 2.0)

KINDS = ("generic", "planar", "mirror", "near_collinear", "collinear", "coincident", "rot180", "identity")
OFFSETS = (0.0, 80.0, 1e3, 1e4)
SPREADS = (1e-3, 0.3, 3.0, 80.0)


def _rot(rng):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q))


def corr_set(kind, n, seed=0, spread=3.0, offset=0.0, inlier_frac=0.6, noise=0.01):
    """-> (ss [n,3] fp32, tt [n,3] fp32, T [4,4] float64: the pose the inliers follow)."""
    rng = np.random.default_rng(seed)
    c = np.array([1.0, -0.5, 0.25]) * offset / np.sqrt(1.3125) if offset else np.zeros(3)
    x = rng.uniform(-1, 1, (n, 3)) * spread
    if kind == "planar":
        x[:, 2] = 0.0
        x = x @ _rot(rng).T
    elif kind == "near_collinear":
        x = np.outer(rng.uniform(-1, 1, n), rng.normal(size=3)) * spread + rng.normal(size=(n, 3)) * 1e-7 * spread
    elif kind == "collinear":
        x = np.zeros((n, 3))
        x[:, 0] = np.round(rng.uniform(-1, 1, n) * spread * 64) / 64
    elif kind == "coincident":
        x = np.zeros((n, 3))
    R = np.eye(3) if kind == "identity" else _rot(rng)
    if kind == "rot180":
        ax = rng.normal(size=3)
        ax /= np.linalg.norm(ax)
        R = 2 * np.outer(ax, ax) - np.eye(3)
    tv = rng.uniform(-1, 1, 3) * min(spread, 1.0)
    s = x + c
    tt = (s - c) @ R.T + c + tv
    if kind == "mirror":
        tt[:, 2] = 2 * c[2] - tt[:, 2]
    tt = tt + rng.normal(scale=noise * min(spread, 1.0), size=(n, 3))
    out = rng.random(n) > inlier_frac
    tt[out] = c + rng.uniform(-1, 1, (int(out.sum()), 3)) * spread
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, c + tv - R @ c
    return s.astype(F32), tt.astype(F32), T


def exact_grid_set(n, offset, seed=0):
    """Correspondences on the fp32 grid of the offset with an exact translation: tt = ss + t0 without rounding, so the
    fp32 and float64 distances of T0 = (I, t0) are both exactly 0 and every weight is 1 on both sides."""
    rng = np.random.default_rng(seed)
    ulp = float(np.spacing(F32(offset))) if offset else 2.0 ** -20
    ss = offset + np.round(rng.uniform(-0.3, 0.3, (n, 3)) / ulp) * ulp
    t0 = np.round(np.array([0.5, -0.25, 0.125]) / ulp) * ulp
    T = np.eye(4)
    T[:3, 3] = t0
    assert (ss.astype(F32) == ss).all() and ((ss + t0).astype(F32) == ss + t0).all()
    return ss.astype(F32), (ss + t0).astype(F32), T


def desc_set(Ka, Kb, seed=0):
    """-> (a [Ka,32], b [Kb,32]) fp32: unit rows with exact duplicates (in b and across a / b), all-zero rows and rows
    one ulp apart."""
    rng = np.random.default_rng(seed)
    a = rng.normal(size=(Ka, 32))
    b = rng.normal(size=(Kb, 32))
    a /= np.linalg.norm(a, axis=1, keepdims=True)
    b /= np.linalg.norm(b, axis=1, keepdims=True)
    a, b = a.astype(F32), b.astype(F32)
    if Kb >= 4:
        b[Kb - 1] = b[1]                      # duplicate across the tile edges
        b[Kb // 2] = b[0]
    if Ka >= 3 and Kb >= 3:
        a[2] = b[Kb // 3]                     # exact match
    for i in range(3, min(Ka, 3 + max(1, Ka // 60))):
        a[i] = 0.0                            # zero descriptors (zero attention)
    if Kb >= 8:
        b[Kb - 3] = 0.0
        b[5] = np.nextafter(b[4], F32(np.inf))  # one ulp apart
    if Ka >= 12 and Kb >= 8:
        a[11] = b[4]
    return np.ascontiguousarray(a), np.ascontiguousarray(b)


def merge(acc, out):
    for k, v in out.items():
        acc[k] = max(acc.get(k, 0.0), v) if isinstance(v, float) else acc.get(k, 0) + v
    return acc


def report(name, out):
    ratios = {k: v for k, v in out.items() if isinstance(v, float)}
    counts = {k: v for k, v in out.items() if isinstance(v, int)}
    print(f"\n[pose-fp64] {name}: " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items())
          + (" | " + ", ".join(f"{k} {v}" for k, v in counts.items()) if counts else ""))


# ------------------------------------------------------------------------------------------------ a10
def _nn_side(M, best, second, got, Kother, what):
    """One side of matching: outside the margin the first float64 minimum; inside it a candidate within the margin, and
    never a later copy of a bitwise-equal row (the first minimum wins on exact ties)."""
    K = M.shape[0]
    if K == 0:
        return 0.0, 0
    eps = lambda d: KN * 35 * U * d + 1e-30
    dec = (second - best) > eps(best) + eps(second)
    ref = M.argmin(1)
    bad = dec & (got != ref)
    assert not bad.any(), f"{what}: decided arg-min differs at {np.flatnonzero(bad)[:5].tolist()}"
    dg = M[np.arange(K), got]
    ratio = (dg - best) / (eps(best) + eps(dg))
    assert (ratio <= 1).all(), f"{what}: pick outside the margin at {np.flatnonzero(ratio > 1)[:5].tolist()}"
    return float(ratio.max(initial=0.0)), int((~dec).sum())


def check_mutual_nn(a, b, snn, tnn, s_mids, t_mids):
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    Ka, Kb = len(a), len(b)
    ref = O.mutual_nn_fp64(a, b)
    out = {}
    if Ka == 0 or Kb == 0:
        assert len(s_mids) == 0
        return dict(matches=0)
    snn, tnn = np.asarray(snn, np.int64), np.asarray(tnn, np.int64)
    out["row_margin"], out["row_marginal"] = _nn_side(ref["D"], ref["r_best"], ref["r_second"], snn, Kb, "row")
    out["col_margin"], out["col_marginal"] = _nn_side(ref["D"].T, ref["c_best"], ref["c_second"], tnn, Ka, "column")
    for M, got, rows, what in ((ref["D"], snn, b, "row"), (ref["D"].T, tnn, a, "column")):
        _, first = np.unique(rows.view(np.int32).reshape(len(rows), -1), axis=0, return_index=True)
        inv = np.unique(rows.view(np.int32).reshape(len(rows), -1), axis=0, return_inverse=True)[1].reshape(-1)
        assert (first[inv[got]] == got).all(), f"{what}: a later copy of an equal row won a tie"
    keep = np.flatnonzero(tnn[snn] == np.arange(Ka))
    assert len(s_mids) == len(keep) and (np.asarray(s_mids) == keep).all() and (np.asarray(t_mids) == snn[keep]).all(), \
        "mutual list is not the ordered mutual set of the arg-mins"
    out["matches"] = len(keep)
    return out


# ------------------------------------------------------------------------------------------------ a13
def check_consensus(ss, tt, R, t, azi_n, inlier_th, counts, best, ind):
    """Each inlier test outside its margin equals float64's; the counts lie in [decided, decided + marginal]; best is
    the first arg-max of the returned counts, with a float64 count interval reaching the largest lower bound; the
    returned inlier list is the best hypothesis's float64 inliers outside the margin."""
    ss, tt, R, t = (np.asarray(x, F32) for x in (ss, tt, R, t))
    Mc = len(ss)
    counts = np.asarray(counts, np.int64)
    if Mc == 0:
        assert len(ind) == 0 and best == 0
        return dict(marginal=0)
    ref = O.consensus_fp64(ss, tt, R, t, azi_n, inlier_th)
    s64, g64 = ss.astype(np.float64), tt.astype(np.float64)
    q_mag = np.abs(R.astype(np.float64)).sum(1) @ np.abs(s64).T + np.abs(t.astype(np.float64)).sum(1)[:, None]
    m = KC * U * (q_mag + np.abs(g64).sum(1)[None] + ref["diffs"] + ref["thr"][None])
    zero = (np.abs(s64).sum(1) == 0)[None]                     # thr = 0 exactly: d < 0 is never true
    marg = (np.abs(ref["diffs"] - ref["thr"][None]) <= m) & ~zero
    lo = (ref["sign"] & ~marg).sum(1)
    hi = (ref["sign"] | marg).sum(1)
    assert ((counts >= lo) & (counts <= hi)).all(), f"counts outside float64's at {np.flatnonzero((counts < lo) | (counts > hi))[:5].tolist()}"
    assert best == int(np.argmax(counts)), "best is not the first arg-max of the counts"
    assert hi[best] >= lo.max(), "best hypothesis cannot reach float64's largest count"
    got = np.zeros(Mc, bool)
    got[np.asarray(ind, np.int64)] = True
    assert (np.diff(np.asarray(ind, np.int64)) > 0).all() and got.sum() == counts[best], "inlier list not ordered / not the count"
    bad = (got != ref["sign"][best]) & ~marg[best]
    assert not bad.any(), f"inlier list differs from float64 outside the margin at {np.flatnonzero(bad)[:5].tolist()}"
    gap = np.abs(ref["diffs"] - ref["thr"][None])
    r = np.where(zero | (m == 0), 0.0, m / np.maximum(gap, 1e-300))
    return dict(marginal=int(marg.sum()), zero_thr=int(zero.sum()) * Mc, decided_min_gap=float(np.where(marg, 0, r).max()))


# ------------------------------------------------------------------------------------------------ a14/a15 fits
def check_fit(a, b, T, what="fit"):
    """A float64 rigid fit of (a, b) against Umeyama: R within bR entrywise (fit_bounds) and t within the lever arm
    3 bR |ca| + KF u53 (|ca| + |cb|).  Degenerate sets: R orthonormal with det 1 and the sum of squared residuals within
    KF u53 of Umeyama's plus the free rotation about the line, which moves no point on it."""
    f = O.fit_bounds(a, b, KF)
    T = np.asarray(T, np.float64)
    R, t = T[:3, :3], T[:3, 3]
    assert np.abs(R @ R.T - np.eye(3)).max() < 1e-12 and np.linalg.det(R) > 0, f"{what}: R is not a rotation"
    if not np.isfinite(f["bR"]):
        a, b = np.asarray(a, np.float64).reshape(-1, 3), np.asarray(b, np.float64).reshape(-1, 3)
        res = ((a @ R.T + t - b) ** 2).sum()
        res64 = ((a @ f["R"].T + f["t"] - b) ** 2).sum()
        scale = (np.abs(a).sum() + np.abs(b).sum()) ** 2
        bound = KF * U53 * scale + 4 * f["off"] * np.sqrt(scale) + 1e-300
        assert res - res64 <= bound, f"{what}: degenerate fit residual {res} above Umeyama's {res64}"
        return dict(deg_res=float(max(res - res64, 0) / bound), degenerate=1)
    eR = np.abs(R - f["R"]).max() / f["bR"]
    bt = 3 * f["bR"] * np.linalg.norm(f["ca"]) + KF * U53 * (np.abs(f["ca"]).sum() + np.abs(f["cb"]).sum())
    et = np.abs(t - f["t"]).max() / bt
    assert eR <= 1 and et <= 1, f"{what}: R {eR:.3g} / t {et:.3g} of the bound from Umeyama"
    return dict(R=float(eR), t=float(et), degenerate=0)


# ------------------------------------------------------------------------------------------------ a14
def check_ransac(src, tgt, ind, dist_th, similar_th, conf, max_iter, seed, T, ninl, bitr, iters, recs=None):
    """One RANSAC run against ransac_fp64: with no marginal decision, (num_inliers, best_itr, iters_run) exactly and T
    within check_fit of Umeyama on the winning triple; otherwise the result is only held to be a valid run (a
    rotation, best_itr < iters_run <= max_iter, a fit of its own triple).  ``recs`` (the C oracle's per-iteration
    records, bit-identical to the kernel's): every decided checker outcome and count equal; a degenerate triple's
    recorded count within its line bound and then taken as the implementation's choice of the free rotation."""
    ref = O.ransac_fp64(src, tgt, ind, dist_th, similar_th, conf, max_iter, seed, kf=KF, recs=recs)
    I = len(ind)
    out = dict(runs=1, decided=0, degenerate_winner=0)
    s = np.asarray(src, F32).astype(np.float64)[np.asarray(ind, np.int64)]
    g = np.asarray(tgt, F32).astype(np.float64)[np.asarray(ind, np.int64)]
    if recs is not None:
        assert len(recs) >= min(iters, ref["iters"])
        for rec in ref["recs"]:
            k = rec["itr"]
            if k >= len(recs) or rec["marginal"]:
                continue
            assert bool(recs["pass"][k]) == rec["passed"], f"itr {k}: checker outcome differs from float64"
            if rec["passed"] and not rec["deg"]:
                assert recs["good"][k] == rec["lo"] == rec["hi"], f"itr {k}: count {recs['good'][k]} vs float64 {rec['lo']}"
    if ref["first_marginal"] is None:
        out["decided"] = 1
        assert (ninl, bitr, iters) == (ref["num_inliers"], ref["best_itr"], ref["iters"]), \
            f"decided run differs: {(ninl, bitr, iters)} vs float64 {(ref['num_inliers'], ref['best_itr'], ref['iters'])}"
    else:
        assert 0 <= iters <= max_iter and bitr < max(iters, 1) and 0 <= ninl <= I
    if bitr >= 0:
        sel = O.ransac_draws(seed, I, bitr + 1)[bitr]
        fit = check_fit(s[sel], g[sel], T, f"best triple {bitr}")
        out["degenerate_winner"] = fit.pop("degenerate")
        out.update({"T_" + k: v for k, v in fit.items()})
    else:
        assert ninl == 0 and np.array_equal(np.asarray(T), np.eye(4)), "no winner: T must be I"
    return out


# ------------------------------------------------------------------------------------------------ a15
def check_refine(src, tgt, T_in, dist_th, T_out, rounds):
    """The refined fp32 pose against refine_fp64.  A round's inlier test is decided when |d64 - th| exceeds the fp32
    evaluation error KD u (|R| |s| + |t| + |g| + d) plus the previous round's fit error moved to the point; with every
    test decided the rounds are equal, R is within KR u + 2 dH / gap and t within KR u |t| + the lever arm 3 bR |ca| +
    the weight shift sum dw |r| / sum w, where a weight moves by dw / w <= 2 (d / th) dd / th + KD u and dH = sum dw |a - ca|
    |r| + KF u53 sum w |a - ca| |b - cb| (r the float64 residual of the fit)."""
    ref = O.refine_fp64(src, tgt, T_in, dist_th)
    s = np.asarray(src, F32).astype(np.float64)
    g = np.asarray(tgt, F32).astype(np.float64)
    th = float(F32(dist_th))
    To = np.asarray(T_out, np.float64).reshape(4, 4)
    assert np.isfinite(To).all()
    Ro = To[:3, :3]
    assert np.abs(Ro @ Ro.T - np.eye(3)).max() < 16 * U and (To[3] == (0, 0, 0, 1)).all()
    bR_prev, bc_prev, ca_prev = 0.0, 0.0, np.zeros(3)
    out = dict(refine_decided=1, refine_marginal=0)
    final = None
    for h in ref["hist"]:
        T = h["T"]
        dd = KD * U * (np.abs(s) @ np.abs(T[:3, :3]).T + np.abs(T[:3, 3]) + np.abs(g)).sum(1) + KD * U * h["d"] \
            + 3 * bR_prev * np.linalg.norm(s - ca_prev, axis=1) + bc_prev
        mg = np.abs(h["d"] - th) <= dd
        if mg.any():
            out["refine_decided"], out["refine_marginal"] = 0, int(mg.sum())
            break
        if "R" not in h:
            break
        m = h["mask"]
        w, a, b = h["w"], s[m], g[m]
        ca, cb = h["cA"], h["cB"]
        r = np.linalg.norm((b - cb) - (a - ca) @ h["R"].T, axis=1)
        dw = w * (2 * (h["d"][m] / th) * dd[m] / th + KD * U)
        da = np.linalg.norm(a - ca, axis=1)
        dH = (dw * da * r).sum() + KF * U53 * (w * da * np.linalg.norm(b - cb, axis=1)).sum()
        d = np.sign(np.linalg.det(h["R"]))
        gap = h["sv"][1] + d * h["sv"][2]
        bR = 2 * dH / gap if gap > 0 else np.inf
        bc = (dw * r).sum() / w.sum() + KF * U53 * (np.abs(ca).sum() + np.abs(cb).sum())
        bR_prev, bc_prev, ca_prev = bR + 2 * U, bc + KD * U * np.abs(h["t"]).sum(), ca
        final = (h, bR, bc)
    if not out["refine_decided"]:
        return out
    assert rounds == ref["rounds"], f"rounds {rounds} vs float64 {ref['rounds']}"
    if final is None:
        assert np.array_equal(To, np.asarray(T_in, F32).astype(np.float64).reshape(4, 4)), "no fit: T must be T_in"
        return out
    h, bR, bc = final
    if not np.isfinite(bR) or bR > 1e-2:
        out["vacuous"] = 1
        return out
    eR = np.abs(Ro - h["R"]).max() / (KR * U + bR)
    bt = KR * U * np.abs(h["t"]).max() + 3 * bR * np.linalg.norm(h["cA"]) + bc
    et = np.abs(To[:3, 3] - h["t"]).max() / bt
    assert eR <= 1 and et <= 1, f"refined pose: R {eR:.3g}, t {et:.3g} of the bound (t off by {np.abs(To[:3, 3] - h['t']).max():.3g} m)"
    out.update(R=float(eR), t=float(et))
    return out
