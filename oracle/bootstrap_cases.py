"""Edge inputs and float64 checks of the loader bootstrap (f1: bx_pca_analysis, bx_project_range,
bx_voxel_down_sample) and of the cpp_wrappers ports (a17 bx_radius_neighbors, a18 bx_grid_subsample), shared by
tests/test_bootstrap_fp64_cpu.py (the oracle, sklearn, the reference's compiled C++) and tests/test_bootstrap_fp64_gpu.py
(the kernels).

The f1 checks hold what a kernel (or the oracle) returned to float64 evaluations of the reference's formulas -- numpy's
``eigh`` of the centred 1/(n-1) covariance, sklearn's PCA itself, ``np.unique`` over float64 voxel tuples -- not to the
oracle's bit contract.  The a17 / a18 checks hold it to the reference's own C++ outputs, stored by
tests/tools/gen_reference_cpp_edges.py in tests/golden/reference_cpp_edges.npz.  The bounds are derived in the
docstring of tests/test_bootstrap_fp64_cpu.py.  Each check returns a dict of ratios (floats, the largest is kept by
``merge``) and counts (ints, summed), printed by ``report``."""
import math
import os

import numpy as np

from oracle.pose_cases import merge  # noqa: F401  (re-exported for the tests)

U24 = 2.0 ** -24
U53 = 2.0 ** -53
F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EDGES_NPZ = os.path.join(ROOT, "tests", "golden", "reference_cpp_edges.npz")
VOXEL_AXIS_CELLS = 1 << 21


def report(name, out):
    ratios = {k: v for k, v in out.items() if isinstance(v, float)}
    counts = {k: v for k, v in out.items() if isinstance(v, (int, np.integer))}
    print(f"\n[bootstrap-fp64] {name}: " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items())
          + (" | " + ", ".join(f"{k} {v}" for k, v in counts.items()) if counts else ""))


def _rot(seed):
    q, r = np.linalg.qr(np.random.default_rng(seed).normal(size=(3, 3)))
    return q * np.sign(np.diag(r))


# ------------------------------------------------------------------------------------------------ f1: PCA clouds
PCA_KINDS = ["generic", "plane", "rod", "disc", "ball", "offset1e5", "offset5e5", "mm", "rot45", "n30"]


def pca_cloud(kind, n=4000, seed=0):
    """-> (fp32 [n,3] cloud, sample indices).  Random clouds take the reference's draw of int(n / 10) indices:
    'generic'; 'plane' (z exactly constant: lambda3 = 0); 'offset1e5' / 'offset5e5' (the generic cloud 1e5 / 5e5 m from
    the origin); 'mm' (1 mm across); 'n30' (30 points: 3 samples).  The exact forms are star clouds sampled in full, so
    that their degeneracies survive fp32: 'rod' (lambda2 = lambda3: z undetermined), 'disc' (lambda1 = lambda2), 'ball'
    (isotropic), 'rot45' (the smallest axis along (1, -1, 0)/sqrt2: the two largest |entries| of the z component tie
    under the sign rule).  The seed scales a star by 2^seed, adds 9 seed repetitions and rolls its axes by seed, all
    exact in fp32, so every seed keeps the degeneracy on other data."""
    rng = np.random.default_rng(seed)
    stars = {"rod": (8.0, 0.3, 0.3, np.eye(3)), "disc": (10.0, 10.0, 0.2, np.eye(3)), "ball": (1.0, 1.0, 1.0, np.eye(3)),
             "rot45": (7.0, 3.0, 0.5, np.array([[1, 0, 1], [1, 0, -1], [0, 1.4142135623730951, 0]]) / 1.4142135623730951)}
    if kind in stars:
        a, b, c, R = stars[kind]
        x = np.roll(star_cloud(a, b, c, R, reps=50 + 9 * seed) * F32(2.0 ** seed), seed, axis=1)
        return x, np.arange(len(x))
    if kind == "n30":
        n = 30
    g = rng.normal(size=(n, 3))
    if kind in ("generic", "offset1e5", "offset5e5", "mm", "n30"):
        x = (g * [6.0, 3.0, 0.4]) @ _rot(seed + 11).T
        x = x * 1e-3 if kind == "mm" else x
        x = x + {"offset1e5": 1e5, "offset5e5": 5e5}.get(kind, 0.0)
    elif kind == "plane":
        x = g * [5.0, 2.0, 0.0] + [0.0, 0.0, 1.5]
    else:
        raise ValueError(kind)
    return x.astype(F32), sample(n, seed)


def sample(n, seed):
    """The reference's draw: np.random.choice(N, int(N / 10), replace=False) from a seeded RandomState."""
    return np.random.RandomState(seed).choice(n, size=int(n / 10), replace=False)


def star_cloud(a, b, c, R=np.eye(3), reps=20, offset=0.0):
    """Repetitions of the six points +-a e1, +-b e2, +-c e3 rotated by R: mean 0, covariance diag(a^2, b^2, c^2) * 2 reps /
    (6 reps - 1) before fp32 rounding.  Sampled in full (the sample indices are an argument of the analysis)."""
    S = np.array([[a, 0, 0], [-a, 0, 0], [0, b, 0], [0, -b, 0], [0, 0, c], [0, 0, -c]], np.float64)
    return (np.tile(S, (reps, 1)) @ R.T + offset).astype(F32)


def margin_pairs():
    """(name, src, tgt, decision) pairs, sampled in full, whose float64 decisions sit a chosen distance from a threshold:
    sphericity vs 0.05, |z . e_z| vs 0.98, dot_z vs 0.96 and round(voxel, 4)'s half-way point, each at relative
    distances 1e-3, 1e-6, 1e-9, 1e-12 on both sides (the smallest lie inside the bounds: they are reported undecided)."""
    out = []
    for d in (1e-3, 1e-6, 1e-9, 1e-12):
        for sgn in (-1, 1):
            t = 1 + sgn * d
            # sphericity = c^2 / a^2 = 0.05 t (b between them); z along e_z exactly, so aligned and same hold
            src = star_cloud(4.0, 2.0, 4.0 * math.sqrt(0.05 * t), reps=24)
            tgt = star_cloud(5.0, 3.0, 1.0)
            out.append((f"sph {sgn * d:+.0e}", src, tgt, "sph"))
            # |z . e_z| = 0.98 t on the source, the target aligned with it
            R = _tilt(math.acos(0.98 * t))
            src = star_cloud(6.0, 3.0, 1.0, R, reps=24)
            tgt = star_cloud(5.0, 2.5, 1.0, R)
            out.append((f"zz {sgn * d:+.0e}", src, tgt, "zz"))
            # dot_z = 0.96 t: both z axes more than 0.98 along e_z, tilted towards opposite sides
            th = math.acos(0.995)
            phi = math.acos(0.96 * t) - th
            src = star_cloud(6.0, 3.0, 1.0, _tilt(th), reps=12)
            tgt = star_cloud(5.0, 2.5, 1.0, _tilt(-phi), reps=10)
            out.append((f"dot {sgn * d:+.0e}", src, tgt, "dot"))
            # voxel = sqrt(2c)/100 (sphericity < 0.05: alpha = 1) at 0.01235 t: round(voxel, 4)'s half-way point
            c = (0.01235 * t * 100) ** 2 / 2
            src = star_cloud(9.0, 8.0, c, reps=12)
            tgt = star_cloud(9.0, 8.0, c, reps=10)
            out.append((f"voxel {sgn * d:+.0e}", src, tgt, "voxel"))
    return out


def _tilt(phi):
    """Rotation about e_y by phi: e_z -> (sin phi, 0, cos phi)."""
    c, s = math.cos(phi), math.sin(phi)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


# ------------------------------------------------------------------------------------------------ f1: float64
def pca_fp64(pts, idx, sklearn=False):
    """eigh of the centred 1/(n-1) covariance of pts[idx] in float64, sorted descending, sklearn's sign rule; with the
    ingredients of the bounds: the covariance entry bound E (n+6) u53 sum|dx_a||dx_b| / (n-1), the eigenvalue bound
    e_lam, per-row gap and component bound e_v (Davis-Kahan, capped at 2), the sign margin of each row.
    sklearn=True widens e_lam for sklearn's own rounding: its covariance_eigh solver forms X^T X - n m m^T without
    centring X, which loses (n + 4) u53 sum|x_a||x_b| / (n - 1) per entry to cancellation far from the origin."""
    X = np.asarray(pts, np.float64)[np.asarray(idx)]
    n = X.shape[0]
    mean = X.mean(0)
    D = X - mean
    C = D.T @ D / (n - 1)
    w, V = np.linalg.eigh(C)
    o = np.argsort(w)[::-1]
    w, V = w[o], V[:, o].T.copy()
    for r in range(3):
        if V[r, np.argmax(np.abs(V[r]))] < 0:
            V[r] = -V[r]
    A = np.abs(D)
    e_mean = (n + 1) * U53 * A.mean(0) + (n + 1) * U53 * np.abs(X).mean(0)
    E = ((n + 6) * U53 * (A.T @ A) + n * np.outer(e_mean, e_mean)) / (n - 1)
    e_lam = 2 * np.linalg.norm(E) + 128 * U53 * np.linalg.norm(C)
    if sklearn:
        e_lam += 2 * np.linalg.norm((n + 4) * U53 * (np.abs(X).T @ np.abs(X)) / (n - 1))
    gap = np.array([min(abs(w[r] - w[s]) for s in range(3) if s != r) for r in range(3)])
    e_v = np.minimum(2.0, 1.5 * e_lam / np.maximum(gap, 1e-300))
    srt = np.sort(np.abs(V), axis=1)
    return dict(mean=mean, var=w, comps=V, e_mean=e_mean, e_lam=e_lam, gap=gap, e_v=e_v,
                sign_margin=srt[:, 2] - srt[:, 1], n=n, absmax=np.abs(X).max(), spread=np.abs(D).max())


def check_pca(pts, idx, mean, var, comps, ref=None):
    """Kernel (or oracle) mean / variances / components against pca_fp64.  Components are checked only where the gap
    determines them (e_v < 0.1), with their sign only where the top two |entries| differ by more than 2 e_v."""
    f = ref or pca_fp64(pts, idx)
    mean, var, comps = (np.asarray(a, np.float64) for a in (mean, var, comps))
    out = {"mean": float((np.abs(mean - f["mean"]) / (2 * f["e_mean"] + 1e-300)).max()),
           "var": float(np.abs(var - f["var"]).max() / f["e_lam"]), "comp": 0.0, "n_comp_undetermined": 0,
           "n_sign_undecided": 0}
    assert out["mean"] <= 1 and out["var"] <= 1, out
    for r in range(3):
        if f["e_v"][r] >= 0.1:
            out["n_comp_undetermined"] += 1
            continue
        assert abs(np.linalg.norm(comps[r]) - 1) <= 1e-12
        g, v = comps[r], f["comps"][r]
        assert g[np.argmax(np.abs(g))] > 0                  # the sign rule on the returned row, first index on a tie
        if f["sign_margin"][r] > 2 * f["e_v"][r]:
            err = np.linalg.norm(g - v)
        else:
            out["n_sign_undecided"] += 1
            err = min(np.linalg.norm(g - v), np.linalg.norm(g + v))
        out["comp"] = max(out["comp"], float(err / f["e_v"][r]))
    assert out["comp"] <= 1, out
    return out


def check_sklearn(pts, idx):
    """pca_fp64 against sklearn's PCA(n_components=3) itself, under the same bounds."""
    from sklearn.decomposition import PCA
    X = np.asarray(pts, np.float64)[np.asarray(idx)]
    p = PCA(n_components=3).fit(X)
    return check_pca(pts, idx, p.mean_, p.explained_variance_, p.components_, ref=pca_fp64(pts, idx, sklearn=True))


def check_range(pts, mean, axis, lo, hi):
    """(lo, hi) of (p - mean) . axis with the kernel's own mean and axis: each side's term within
    4 u53 max_i sum_c |p_ic - m_c||a_c| of the exact value (a difference, a product, two sums), 10 u53 for the pair."""
    P = np.asarray(pts, np.float64)
    m, a = np.asarray(mean, np.float64), np.asarray(axis, np.float64)
    z = (P - m) @ a
    e = 10 * U53 * (np.abs(P - m) @ np.abs(a)).max() + 1e-300
    return {"range": float(max(abs(lo - z.min()), abs(hi - z.max())) / e)}


def reference_analysis(src, tgt, idx_s, idx_t):
    """sphericity_based_voxel_analysis (utils/tools.py:132-198) evaluated with sklearn's PCA, float64 throughout
    (Open3D points are doubles), and the float64 ingredients of the decision margins."""
    from sklearn.decomposition import PCA
    res = []
    for pts, idx in ((src, idx_s), (tgt, idx_t)):
        P = np.asarray(pts, np.float64)
        p = PCA(n_components=3).fit(P[np.asarray(idx)])
        z = p.components_[-1] / np.linalg.norm(p.components_[-1])
        res.append(dict(pca=p, sph=p.explained_variance_[2] / p.explained_variance_[0], zz=abs(z[2]), z=z,
                        f=pca_fp64(pts, idx, sklearn=True), P=P))
    s, t = res
    ref = s if len(src) > len(tgt) else t
    zr = ref["pca"].transform(ref["P"])[:, 2]
    z_range = zr.max() - zr.min()
    alpha = 1.0 if ref["sph"] < 0.05 else 1.5
    voxel = max(np.sqrt(z_range) / 100 * alpha, 0.001)
    dot = float(np.dot(s["z"], t["z"]))
    return dict(voxel=round(float(voxel), 4), sph=float(ref["sph"]), aligned=bool(s["zz"] > 0.98 and t["zz"] > 0.98 and dot > 0.96),
                raw_voxel=float(voxel), z_range=float(z_range), alpha=alpha, dot=dot, s=s, t=t, ref=ref)


def check_analysis(got, rf):
    """(voxel, sphericity, is_aligned) of the kernel route against reference_analysis.  A decision is compared where its
    float64 margin exceeds its bound; the others are counted (``undecided_*``) and listed with their margins."""
    voxel, sph, aligned = got
    ref = rf["ref"]
    f = ref["f"]
    lam1 = f["var"][0]
    e_sph = f["e_lam"] * (1 + rf["sph"]) / lam1
    out = {"sph": float(abs(sph - rf["sph"]) / e_sph), "undecided": [], "closest": 0.0}

    def decided(margin, e):                   # closest: the largest bound / margin among the decided decisions
        if abs(margin) > e:
            out["closest"] = max(out["closest"], float(e / abs(margin)))
            return True
        return False

    assert out["sph"] <= 1, (sph, rf["sph"], e_sph)
    # the z-range moves with the axis (e_v of row 2 times the spread) and the projection's rounding
    e_zr = 4 * math.sqrt(3) * f["spread"] * f["e_v"][2] + 36 * U53 * f["absmax"]
    sph_dec = decided(rf["sph"] - 0.05, e_sph)
    zr = max(rf["z_range"], 1e-300)
    e_vox = rf["alpha"] * e_zr / (200 * math.sqrt(zr)) + 8 * U53
    half = (math.floor(rf["raw_voxel"] * 1e4) + 0.5) * 1e-4
    vox_dec = sph_dec and f["e_v"][2] < 0.1 and decided(rf["raw_voxel"] - half, e_vox)
    if vox_dec:
        assert voxel == rf["voxel"], (voxel, rf)
    else:
        out["undecided"].append(("voxel", rf["raw_voxel"] - half, e_vox))
    # aligned = |zs_z| > 0.98 and |zt_z| > 0.98 and zs . zt > 0.96, three-valued
    parts = []
    for c in (rf["s"], rf["t"]):
        e = c["f"]["e_v"][2] + 4 * U53
        parts.append(bool(c["zz"] > 0.98) if decided(c["zz"] - 0.98, e) else None)
        if parts[-1] is None:
            out["undecided"].append(("zz", c["zz"] - 0.98, e))
    e_dot = rf["s"]["f"]["e_v"][2] + rf["t"]["f"]["e_v"][2] + 8 * U53
    signs = all(c["f"]["sign_margin"][2] > 2 * c["f"]["e_v"][2] for c in (rf["s"], rf["t"]))
    parts.append(bool(rf["dot"] > 0.96) if signs and decided(rf["dot"] - 0.96, e_dot) else None)
    if parts[-1] is None:
        out["undecided"].append(("dot", rf["dot"] - 0.96, e_dot))
    dec = False if False in parts else (True if all(p is True for p in parts) else None)
    if dec is not None:
        assert aligned == dec, (aligned, rf["aligned"], parts)
        assert rf["aligned"] == dec
    out["n_undecided"] = len(out["undecided"])
    return out


# ------------------------------------------------------------------------------------------------ f1: voxel down-sampling
VDS_KINDS = ["gauss", "kvoxel", "same", "one", "negoff", "dense"]


def vds_cloud(kind, seed=0):
    """-> (fp32 cloud, voxel).  'kvoxel': points exactly k voxel from voxel_min_bound and one fp32 ulp either side,
    for a dyadic voxel (exact) and 0.035; 'same': 5000 identical points; 'one': n = 1; 'negoff': negative coordinates
    -3e3 m and beyond; 'dense': 1e5 points in one voxel (the fp64 atomic mean)."""
    rng = np.random.default_rng(seed)
    if kind == "gauss":
        return (rng.normal(size=(20000, 3)) * [8.0, 5.0, 1.5]).astype(F32), 0.035
    if kind == "kvoxel":
        voxel = 0.25 if seed % 2 == 0 else 0.035
        vmb = 0.0 - voxel * 0.5
        k = rng.integers(1, 60, (3000, 3))
        x = (vmb + k * voxel).astype(F32)
        step = rng.integers(-1, 2, x.shape)
        x = np.where(step < 0, np.nextafter(x, F32(-np.inf)), np.where(step > 0, np.nextafter(x, F32(np.inf)), x))
        return np.concatenate([np.zeros((1, 3), F32), x]).astype(F32), voxel
    if kind == "same":
        return np.tile(np.array([[1.25, -3.5, 7.0]], F32), (5000, 1)), 0.05
    if kind == "one":
        return np.array([[-2.5, 3.25, 1e3]], F32), 0.3
    if kind == "negoff":
        return (rng.normal(size=(8000, 3)) * [30.0, 20.0, 2.0] - [3e3, 4e4, 1e2]).astype(F32), 0.3
    if kind == "dense":
        return (rng.uniform(0, 0.01, (100000, 3)) + [123.0, -45.0, 6.0]).astype(F32), 1.0
    raise ValueError(kind)


def vds_fp64(P, voxel):
    """Open3D's VoxelDownSample in float64: (tuples [m,3] int64 sorted, means [m,3] float64, counts [m], inverse)."""
    P = np.asarray(P, np.float64)
    vmb = P.min(0) - voxel * 0.5
    iv = np.floor((P - vmb) / voxel).astype(np.int64)
    t, inv, cnt = np.unique(iv, axis=0, return_inverse=True, return_counts=True)
    inv = inv.reshape(-1)
    s = np.zeros((len(t), 3))
    np.add.at(s, inv, P)
    return t, s / cnt[:, None], cnt, inv


def check_vds(pts, voxel, keys, xyz, cnt):
    """Kernel keys against an independent (ix, iy, iz) tuple from np.unique(axis=0) (not the oracle's masked key),
    counts exactly, means within u24 |mean| (fp32 output) + (cnt + 2) u53 max|p| (fp64 sums in any order)."""
    t, mean, c, _ = vds_fp64(pts, voxel)
    keys = np.asarray(keys).astype(np.int64)
    tk = np.stack([keys & 0x1FFFFF, (keys >> 21) & 0x1FFFFF, (keys >> 42) & 0x1FFFFF], 1)
    o = np.lexsort((tk[:, 2], tk[:, 1], tk[:, 0]))
    assert len(keys) == len(t) and np.array_equal(tk[o], t), "voxel sets differ"
    assert np.array_equal(np.asarray(cnt)[o], c)
    e = U24 * np.abs(mean) + (c[:, None] + 2) * U53 * np.abs(np.asarray(pts, np.float64)).max() + 1e-300
    r = float((np.abs(np.asarray(xyz, np.float64)[o] - mean) / e).max())
    assert r <= 1, r
    return {"mean": r, "n_voxels": len(t)}


def check_reassigned(t64, t_k, e):
    """t64 / t_k: the float64 and the kernel-side cell coordinates (p - vmb) / voxel [m,3]; e [m,3] the bound of their
    difference.  Every point in a different cell must lie within e of a cell boundary on each axis that differs."""
    f64, fk = np.floor(t64), np.floor(t_k)
    diff = f64 != fk
    dist = np.abs(t64 - np.round(t64))
    r = float((dist[diff] / e[diff]).max()) if diff.any() else 0.0
    assert r <= 1, (r, np.argwhere(diff)[:5])
    assert (np.abs(f64 - fk) <= 1).all()
    return {"reassign": r, "n_reassigned": int(diff.any(1).sum())}


def check_loader_route(P_in, downsample, voxel0, first, second):
    """The loader's two calls: voxel_down_sample(downsample), then voxel_down_sample(voxel0) on its output.  ``first`` /
    ``second`` are the kernel's (keys, fp32 means, counts) of each call (the second on the first's fp32 means).  The
    first call is exact against float64; the second's input differs from Open3D's float64 means by their fp32 rounding
    and fp64 summation, so a first-stage voxel may change second-stage cell only within that of a cell boundary."""
    out = check_vds(np.asarray(P_in, F32), downsample, *first)
    P = np.asarray(P_in, F32).astype(np.float64)
    t1, m64, c1, _ = vds_fp64(P, downsample)
    keys, xyz, cnt = (np.asarray(a) for a in first)
    keys = keys.astype(np.int64)
    tk = np.stack([keys & 0x1FFFFF, (keys >> 21) & 0x1FFFFF, (keys >> 42) & 0x1FFFFF], 1)
    o = np.lexsort((tk[:, 2], tk[:, 1], tk[:, 0]))
    mk = np.asarray(xyz, np.float64)[o]                         # the kernel's means, in float64's voxel order
    dm = U24 * np.abs(m64) + (c1[:, None] + 2) * U53 * np.abs(P).max()
    vmb64 = m64.min(0) - voxel0 * 0.5
    vmbk = mk.min(0) - voxel0 * 0.5
    e = (dm + dm.max(0)) / voxel0 * 1.01 + 4 * U53 * (np.abs(m64) / voxel0 + 1)
    merge(out, check_reassigned((m64 - vmb64) / voxel0, (mk - vmbk) / voxel0, e))
    out2 = check_vds(np.asarray(xyz, F32), voxel0, *second)
    out["mean2"] = out2["mean"]
    return out


def check_fp64_input(P64, voxel, keys, xyz, cnt):
    """float64 input to bootstrap.voxel_down_sample, which rounds it to fp32 first: the kernel is exact on the rounded
    cloud, and every point assigned differently from Open3D on the doubles lies within fp32 rounding of a boundary."""
    P32 = np.asarray(P64, F32)
    out = check_vds(P32, voxel, keys, xyz, cnt)
    P64 = np.asarray(P64, np.float64)
    P = P32.astype(np.float64)
    e = (np.abs(P - P64) + np.abs(P.min(0) - P64.min(0))) / voxel * 1.01 + 4 * U53 * (np.abs(P64) / voxel + 1)
    merge(out, check_reassigned((P64 - (P64.min(0) - voxel * 0.5)) / voxel, (P - (P.min(0) - voxel * 0.5)) / voxel, e))
    return out


def analysis_pairs():
    """(name, src, tgt, idx_src, idx_tgt): generic pairs, ns == nt (the reference takes the target), ns > nt, the
    degenerate clouds and the decision-margin pairs (sampled in full)."""
    out = []
    (g0, i0), (g1, i1) = pca_cloud("generic", 4000, 0), pca_cloud("generic", 4000, 1)
    out.append(("ns==nt", g0, g1, i0, i1))
    (r, ir), (d, idd) = pca_cloud("rod"), pca_cloud("disc")
    out.append(("rod vs disc", r, d, ir, idd))
    (b, ib), (t, it) = pca_cloud("ball"), pca_cloud("rot45")
    out.append(("ball vs rot45", t, b[:-6], it, ib[:-6]))
    (p, ip), (o, io) = pca_cloud("plane", 3000, 4), pca_cloud("offset5e5", 6000, 5)
    out.append(("plane<offset5e5", p, o, ip, io))
    for name, s, t, _ in margin_pairs():
        out.append((name, s, t, np.arange(len(s)), np.arange(len(t))))
    return out


def axis_limit_cloud(voxel):
    """Two points whose x extent puts the top index at 2^21 - 1 exactly, and the same with the next fp32 coordinate
    (index 2^21)."""
    top = lambda x: math.floor((float(x) - (0.0 - voxel * 0.5)) / voxel)
    x = np.float32((VOXEL_AXIS_CELLS - 0.75) * voxel)
    while top(x) >= VOXEL_AXIS_CELLS:
        x = np.nextafter(x, np.float32(0))
    while top(np.nextafter(x, np.float32(np.inf))) < VOXEL_AXIS_CELLS:
        x = np.nextafter(x, np.float32(np.inf))
    inside = np.array([[0, 0, 0], [x, 1, 1]], np.float32)
    beyond = np.array([[0, 0, 0], [np.nextafter(x, np.float32(np.inf)), 1, 1]], np.float32)
    assert top(inside[1, 0]) == VOXEL_AXIS_CELLS - 1 and top(beyond[1, 0]) == VOXEL_AXIS_CELLS
    return inside, beyond


def loader_clouds():
    """(name, cloud, downsample): clouds for the loader's two calls, with the voxel their analysis gives."""
    out = []
    for name, kind, n, seed in (("generic", "generic", 30000, 0), ("offset1e5", "offset1e5", 20000, 1)):
        pts, _ = pca_cloud(kind, n, seed)
        rf = reference_analysis(pts, pts, sample(n, seed), sample(n, seed + 1))
        out.append((name, pts, rf["voxel"]))
    return out


# ------------------------------------------------------------------------------------------------ a17 / a18 edge inputs
def _lattice(k, step=1.0, offset=0.0):
    g = np.stack(np.meshgrid(*[np.arange(k)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float64)
    return ((g - (k - 1) / 2) * step + offset).astype(F32)


R_SQRT5 = F32(np.sqrt(5.0))          # fl32(r * r) == 5 exactly, although r^2 = 5.00000015 in float64
assert F32(R_SQRT5 * R_SQRT5) == 5.0 and float(R_SQRT5) ** 2 > 5.0


def neighbor_cases():
    """name -> (queries, supports, q_batches, s_batches, radius).  Lattices give exact distance ties; 'ball4096' has
    more than 4096 entries per ball (the global rank sort); 'sqrt5' and 'r2' put lattice points exactly on the strict
    boundary d = fl32(r * r); 'empty' has no neighbour at all (mc = 0); 'b1' ... 'b8' are 1 to 8 query batches over two
    support clouds (odd batches search cloud 1); 'offset' sits 1e3 m from the origin."""
    rng = np.random.default_rng(17)
    out = {}
    L9 = _lattice(9, 0.1)
    q = L9[rng.choice(len(L9), 200, replace=False)]
    for r in (0.15, 0.25, 0.35):
        out[f"lat9_{r}"] = (q, L9, [200], [len(L9)], r)
    L23 = _lattice(23)
    qc = np.concatenate([_lattice(3), _lattice(2) + F32(0.5), np.array([[0.25, -0.5, 0.125]], F32)]).astype(F32)
    out["ball4096"] = (qc, L23, [len(qc)], [len(L23)], 10.5)
    L7 = _lattice(7)
    out["sqrt5"] = (L7[::5], L7, [len(L7[::5])], [len(L7)], float(R_SQRT5))
    out["r2"] = (L7[::3], L7, [len(L7[::3])], [len(L7)], 2.0)
    out["empty"] = (L7[:40] + F32(100.0), L7, [40], [len(L7)], 0.9)
    s0 = _lattice(6, 0.5)
    s1 = (rng.uniform(-1.5, 1.5, (300, 3))).astype(F32)
    sup = np.concatenate([s0, s1])
    for nb in (1, 2, 3, 8):
        qb = [int(v) for v in rng.integers(1, 30, nb)]
        qs = []
        for b, m in enumerate(qb):
            src = s0 if b % 2 == 0 else s1
            qs.append(src[rng.choice(len(src), m, replace=False)] + F32(0.01) * (b % 3))
        out[f"b{nb}"] = (np.concatenate(qs).astype(F32), sup, qb, [len(s0), len(s1)] if nb > 1 else [len(s0)], 0.55)
    Lo = _lattice(8, 0.25, 1e3)
    out["offset"] = (Lo[rng.choice(len(Lo), 100, replace=False)], Lo, [100], [len(Lo)], 0.3)
    return out


def origin_above_min(dl, lo):
    """First fp32 m among lo, lo + 1e-3, ... with floorf(m * (1/dl)) * dl > m (the grid origin rounds above the minimum)."""
    dl = F32(dl)
    inv = F32(1) / dl
    for k in range(1000):
        m = F32(lo + 1e-3 * k)
        if F32(np.floor(F32(m * inv)) * dl) > m:
            return m
    raise ValueError("no such minimum")


def subsample_cases():
    """name -> (points, dl).  'above_x' / 'above_y': the fp32 origin rounds above the minimum on x / y, and the point
    at the minimum corner gets cell -1 on that axis -- its key wraps to 2^64 - 1 ('above_x': cell (-1, 0, 0)) or to
    the row below ('above_y'); 'offset1e3': 1e3 m from the origin; 'lattice': dyadic points exactly on cell faces;
    'uniform' a generic cloud; 'flat_x' / 'flat_y': every x (y) equals such a minimum, so the reference's NX (NY) is 0
    and whole rows of cells alias -- 'flat_x' is one cell; 'pair_y': two points on it that differ only in y, one cell."""
    rng = np.random.default_rng(23)
    out = {}
    dl = 0.025
    m = float(origin_above_min(dl, 40.6))
    edge = np.concatenate([np.full((20, 1), m), rng.uniform(0, 0.3, (20, 2))], 1)   # cell -1 on x: aliased cells
    p = rng.uniform(0, 0.3, (3000, 3)) + [m, 0.0, 0.0]
    p = np.concatenate([[[m, 0.0, 0.0]], edge, p]).astype(F32)
    out["above_x"] = (p, dl)
    p = rng.uniform(0, 0.3, (3000, 3)) + [0.0, m, 0.0]
    p = np.concatenate([[[0.3, m, 0.0]], p]).astype(F32)
    p[1:, 0] = np.minimum(p[1:, 0], F32(0.3))
    out["above_y"] = (p, dl)
    out["offset1e3"] = ((rng.uniform(-3, 3, (8000, 3)) * [1, 1, 0.4] + 1e3).astype(F32), 0.1)
    out["lattice"] = (_lattice(16, 0.125, 0.0625), 0.25)
    out["uniform"] = ((rng.uniform(-3, 3, (8000, 3)) * [1, 1, 0.4]).astype(F32), 0.2)
    # flat axes at the rounded-up origin: floor((max - origin) / dl) = -1 gives NX = 0 (NY = 0), so every key aliases
    rng = np.random.default_rng(29)
    p = rng.uniform(0, 0.3, (500, 3))
    p[:, 0] = m
    out["flat_x"] = (p.astype(F32), dl)
    p = rng.uniform(0, 0.3, (500, 3))
    p[:, 1] = m
    out["flat_y"] = (p.astype(F32), dl)
    out["pair_y"] = (np.array([[m, 0.0, 0.0], [m, 0.1, 0.0]], F32), dl)
    return out


# ------------------------------------------------------------------------------------------------ a17 / a18 checks
def row_distances(q, s, row):
    """float64 squared distances of the listed entries of one row (the reference's d from the fp32 coordinates)."""
    d = np.asarray(s, np.float64)[row] - np.asarray(q, np.float64)
    return ((d[:, 0] * d[:, 0]) + (d[:, 1] * d[:, 1])) + (d[:, 2] * d[:, 2])


def check_neighbors(q, s, qb, sb, radius, got, ref=None, oracle_rows=None):
    """Rows of ``got`` against the reference's: the same distance sequence exactly and, inside every run of equal
    distance, the same index set; against the oracle's (distance, index) order exactly.  Also float64 ground truth:
    every listed entry has d < fl32(r * r), no other support of the searched cloud does."""
    got = np.asarray(got)
    ns = len(s)
    r2 = float(F32(F32(radius) * F32(radius)))
    out = {"n_tie_rows": 0, "n_rows": len(got)}
    if ref is not None:
        assert got.shape == ref.shape, (got.shape, ref.shape)
    if oracle_rows is not None:
        assert got.shape == oracle_rows.shape and np.array_equal(got, oracle_rows)
    acc = np.concatenate([[0], np.cumsum(qb)])
    for i in range(len(got)):
        b = int(np.searchsorted(acc, i, side="right") - 1)
        off, n = (0, sb[0]) if b % 2 == 0 else (sb[0], sb[1])
        row = got[i][got[i] != ns]
        assert (got[i][len(row):] == ns).all()
        d = row_distances(q[i], s, row)
        assert (d < r2).all() and ((row >= off) & (row < off + n)).all()
        assert (np.diff(d) >= 0).all() and all(row[k] < row[k + 1] for k in range(len(row) - 1) if d[k] == d[k + 1])
        dall = row_distances(q[i], s, np.arange(off, off + n))
        assert (dall < r2).sum() == len(row)
        if ref is not None:
            rr = ref[i][ref[i] != ns]
            dr = row_distances(q[i], s, rr)
            assert np.array_equal(d, dr), i
            if not np.array_equal(rr, row):
                out["n_tie_rows"] += 1
                _, starts = np.unique(d, return_index=True)
                for a, z in zip(starts, list(starts[1:]) + [len(d)]):
                    assert set(rr[a:z].tolist()) == set(row[a:z].tolist()), i
    return out


def bary_bound(xyz, cnt, dl):
    """(cnt + 2) u24 max|p| per coordinate: fp32 sums in any order (cnt - 1 additions), fl32(1 / cnt) and the product,
    with max|p| <= max|barycentre| + 2 dl (a cell is dl wide; an aliased cell spans the cloud's x extent, bounded
    here by the magnitude of the barycentre's cloud)."""
    xyz = np.abs(np.asarray(xyz, np.float64))
    return (np.asarray(cnt, np.float64)[:, None] + 2) * U24 * (xyz.max() + 2 * dl)


def _bitsort(x):
    x = np.ascontiguousarray(x, F32)
    return x[np.lexsort((x[:, 2], x[:, 1], x[:, 0]))]


def check_subsample(pts, dl, keys, xyz, cnt, ref_xyz, oracle_out):
    """Kernel cells against the oracle's (keys and counts exactly; barycentres within twice bary_bound, both summing in
    their own order) and against the reference's barycentre set (the same number of cells; the oracle's barycentres are
    the reference's bit for bit)."""
    ek, exyz, ecnt = oracle_out
    k = np.asarray(keys).astype(np.uint64)
    o = np.argsort(k, kind="stable")
    assert len(k) == len(ref_xyz) == len(ek), (len(k), len(ref_xyz), len(ek))
    assert np.array_equal(k[o], ek) and np.array_equal(np.asarray(cnt)[o], ecnt)
    assert int(np.asarray(cnt).sum()) == len(pts)
    assert np.array_equal(_bitsort(exyz), _bitsort(ref_xyz)), "oracle barycentres != reference barycentres"
    e = 2 * bary_bound(exyz, ecnt, dl)
    r = float((np.abs(np.asarray(xyz, np.float64)[o] - exyz) / e).max())
    assert r <= 1, r
    return {"bary": r, "n_cells": len(k), "n_wrapped": int((ek > np.uint64(1 << 63)).sum())}


def load_edges():
    with np.load(EDGES_NPZ) as z:
        return {k: z[k] for k in z.files}
