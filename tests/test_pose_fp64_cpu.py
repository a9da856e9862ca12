"""Mutual matching, consensus, RANSAC and refinement (a10, a13-a15) against float64 without a GPU: the C oracle's
bxo_mutual_nn, bxo_consensus, horn_fit, bxo_ransac (iteration by iteration, through its records) and bxo_refine held to
the float64 evaluations of oracle.py (mutual_nn_fp64, consensus_fp64, umeyama_fp64, ransac_fp64, refine_fp64), which
restate the reference's formulas (knn, BUFFERX.py:404-417, Open3D's point-to-point estimation and RANSAC loop,
post_refinement + rigid_transform_3d) rather than the C code.  The kernels are held bit for bit to the same oracle and
to the same checks in tests/test_pose_fp64_gpu.py.

The bounds (oracle/pose_cases.py; u = 2^-24, u53 = 2^-53):

* Matching.  fl32(d) = sum_c fl(a_c - b_c)^2 over C = 32 terms is within (C + 3) u d of the float64 distance (every term
  is non-negative, so the sum's error is relative to d itself).  A row's arg-min is decided when the float64 gap between
  the best and the second best exceeds the two errors (KN = 4 of slack); a decided arg-min must be float64's, an
  undecided one must lie within the margin of the minimum.  Bitwise-equal rows give bitwise-equal fp32 distances, so
  among them the first index must win (knn's tie rule), and the mutual list is the ordered set with tnn[snn[i]] = i.
* Consensus.  q = R s + t, q - g, the norm and thr = |s| pi / azi_n * inlier_th in fp32 are each within a few u of
  their magnitudes: |fl(d) - d64| + |fl(thr) - thr64| <= KC u (|R| |s| + |t| + |g| + d + thr).  Outside that margin the
  inlier test equals float64's (d < thr, strict); a key point at the origin has thr = 0 exactly and is never an
  inlier.  Counts lie in [decided inliers, decided + marginal]; best is the first arg-max of the counts.
* Fits.  A float64 fit of H = sum w (a - ca)(b - cb)^T perturbed by dH moves R by <= 2 |dH| / (sigma_2 + d sigma_3)
  (the conditioning of the polar factor with the det correction d = +-1; kappa = sigma_1 / (sigma_2 + d sigma_3)).
  Rounding in float64 gives |dH| <= KF u53 sum w |a - ca| |b - cb| -- the centred magnitudes, so a fit that cancels an
  offset^2 (an uncentred cross-covariance) fails far from the origin.  t = cb - R ca: within the lever arm 3 bR |ca| plus
  the centroid rounding.  Where the bound exceeds 1e-6 (collinear, duplicate or coincident points) the rotation about
  the line is free: the fit's residual is held to Umeyama's instead.
* RANSAC.  Each iteration's checkers and inlier tests are decided outside the fit margin (3 bR |x - ca| plus rounding);
  a degenerate triple's count lies in [0, hi], hi the correspondences within dist_th of the target line in cylinder
  coordinates, and is decided only once hi is below the best count.  A run without a marginal decision must give
  (num_inliers, best_itr, iters_run) exactly and T within the fit bound of the winning triple.
* Refinement.  The fp32 distances are within KD u (|R| |s| + |t| + |g| + d) plus the previous round's fit error;
  weights move by dw / w <= 2 (d / th) dd / th + KD u, and only through the fit residual r do they rotate R (a symmetric
  change of H leaves the polar factor alone): dH = sum dw |a - ca| |r| + KF u53 sum w |a - ca| |b - cb|.  R within
  KR u + 2 dH / gap, t within KR u |t| + 3 bR |ca| + sum dw |r| / sum w.  Both sides use the reference's centroids over
  (sum w + 1e-6).  The exact-grid cases (every distance exactly 0 in fp32 and float64) make the weights equal, so far
  from the origin only the float64 rounding of the fit remains.

The largest ratios are printed with -s and recorded in DESIGN.md section 7."""
import numpy as np
import pytest

from oracle import pose_cases as P
from oracle.pose_cases import merge, report

KAB = [1, 63, 64, 65, 1023, 1024, 1025, 1500]


def test_philox_against_published_vectors_and_oracle(oracle):
    """Philox4x32-10 known-answer vectors (Salmon et al., Random123) and the oracle's per-iteration draws: a RANSAC run
    whose records equal the float64 replay's iteration by iteration (checked below) only follows the same draws."""
    from oracle.oracle import philox4x32_10_np
    kat = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
           ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
           ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
            (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in kat:
        assert tuple(int(x) for x in philox4x32_10_np(np.array([ctr], np.uint64), key)[0]) == want
    sel = oracle.ransac_draws(0x123456789, 7, 5)
    assert sel.shape == (5, 3) and (sel >= 0).all() and (sel < 7).all()


@pytest.mark.parametrize("Ka", KAB)
def test_mutual_nn_vs_fp64(oracle, Ka):
    acc = {}
    for Kb in KAB:
        a, b = P.desc_set(Ka, Kb, seed=Ka + Kb)
        s, t, snn, tnn = oracle.mutual_nn(a, b)
        merge(acc, P.check_mutual_nn(a, b, snn, tnn, s, t))
    report(f"mutual_nn Ka={Ka}, every Kb", acc)


@pytest.mark.parametrize("inlier_th", P.INLIER_TH)
@pytest.mark.parametrize("n", [0, 1, 3, 257, 1025])
def test_consensus_vs_fp64(oracle, n, inlier_th):
    acc = {}
    for k, kind in enumerate(P.KINDS):
        ss, tt, T = P.corr_set(kind, n, seed=n + k, offset=P.OFFSETS[k % 4] if kind == "generic" else 0.0)
        rng = np.random.default_rng(k)
        R = np.tile(T[:3, :3].astype(np.float32), (n, 1, 1))
        t = (T[:3, 3] + rng.normal(scale=0.05, size=(n, 3))).astype(np.float32)
        if n >= 3:
            ss[0] = 0.0                                    # thr = 0 exactly ...
            t[1] = tt[0]                                   # ... and d = 0 exactly for hypothesis 1
            R[2::3] = np.eye(3, dtype=np.float32)
        ind, best, counts = oracle.consensus(ss, tt, R, t, 20, inlier_th)
        merge(acc, P.check_consensus(ss, tt, R, t, 20, inlier_th, counts, best, ind))
    report(f"consensus n={n} inlier_th={inlier_th:.3g}", acc)


@pytest.mark.parametrize("kind", P.KINDS)
def test_horn_fit_vs_umeyama(oracle, kind):
    acc = {}
    for spread in P.SPREADS:
        for offset in P.OFFSETS:
            for n in (3, 4, 256):
                ss, tt, _ = P.corr_set(kind, n, seed=n, spread=spread, offset=offset, inlier_frac=1.0)
                a, b = ss.astype(np.float64), tt.astype(np.float64)
                merge(acc, P.check_fit(a, b, oracle.horn_fit(a, b), f"{kind} spread {spread} offset {offset} n {n}"))
    report(f"horn_fit {kind}", acc)


RANSAC_RUNS = [(n, kind, dt, st) for n in (3, 4, 255, 1023, 4500) for kind in ("generic", "planar", "collinear", "identity")
               for dt, st in ((0.10, 0.8), (0.30, 0.9))]


@pytest.mark.parametrize("n,kind,dist_th,similar_th", RANSAC_RUNS)
def test_ransac_per_iteration_vs_fp64(oracle, n, kind, dist_th, similar_th):
    ss, tt, _ = P.corr_set(kind, n + 20, seed=n, inlier_frac=0.5)
    ind = np.arange(n, dtype=np.int32)
    acc = {}
    for conf, iters in ((0.999, 5000), (1.0, 300)):
        r = oracle.ransac(ss, tt, ind, dist_th, similar_th, conf, iters, 77, want_recs=True)
        merge(acc, P.check_ransac(ss, tt, ind, dist_th, similar_th, conf, iters, 77, r["T"], r["num_inliers"],
                                  r["best_itr"], r["iters"], recs=r["recs"]))
    report(f"ransac n={n} {kind} dist_th={dist_th}", acc)


def test_ransac_all_inliers_stops_at_once(oracle):
    """Every correspondence an inlier: r = 1, est_k = ceil(-0.0) = 0, the loop ends after the first winner."""
    ss, tt, _ = P.corr_set("generic", 300, seed=3, inlier_frac=1.0, noise=0.0)
    ind = np.arange(300, dtype=np.int32)
    r = oracle.ransac(ss, tt, ind, 0.10, 0.8, 0.999, 1000, 5, want_recs=True)
    out = P.check_ransac(ss, tt, ind, 0.10, 0.8, 0.999, 1000, 5, r["T"], r["num_inliers"], r["best_itr"], r["iters"], recs=r["recs"])
    assert out["decided"] and r["num_inliers"] == 300 and r["iters"] == r["best_itr"] + 1


REFINE = [(kind, off, dt) for kind in ("generic", "planar", "identity", "rot180") for off in (0.0, 80.0) for dt in P.DIST_TH]


@pytest.mark.parametrize("kind,offset,dist_th", REFINE)
def test_refine_vs_fp64(oracle, kind, offset, dist_th):
    ss, tt, T = P.corr_set(kind, 900, seed=4, spread=3.0, offset=offset, inlier_frac=0.6, noise=0.01)
    T0 = T.copy()
    T0[:3, 3] += 0.3 * dist_th
    To, rounds = oracle.refine(ss, tt, T0.astype(np.float32), dist_th)
    out = P.check_refine(ss, tt, T0, dist_th, To, rounds)
    report(f"refine {kind} offset {offset} dist_th {dist_th}", out)


@pytest.mark.parametrize("offset", [0.0, 80.0, 1e3, 1e4])
def test_refine_exact_grid_far_from_origin(oracle, offset):
    """Every distance exactly 0: the weights are 1 on both sides and the bound is the fit's float64 rounding, so an
    uncentred cross-covariance (offset^2 cancellation) fails at 1e4 m."""
    ss, tt, T = P.exact_grid_set(900, offset, seed=1)
    To, rounds = oracle.refine(ss, tt, T.astype(np.float32), 0.10)
    out = P.check_refine(ss, tt, T, 0.10, To, rounds)
    assert out["refine_decided"] and "R" in out
    report(f"refine exact grid offset {offset:g}", out)
