"""FPS, radius estimation and patch gathering (a1-a3) against float64 without a GPU: the C oracle's bxo_fps,
bxo_radius_hist / bxo_radius_bisect (with radius_estimation's cloud choice, sub-sampling and rounding), bxo_ball_query
and bxo_select_patches held to the float64 evaluations of oracle.py (fps_fp64, radius_count_bounds / radius_fp64 /
radius_replay, ball_query_fp64, select_patches_fp64).  Those restate the reference's formulas (pointnet2's
furthest_point_sample and ball_query, squared_cdist + the bisection of BUFFERX.py:627-696, the mask rules of
patch_embedder.py:92-120) rather than the C code, so an error made on both sides of the bit contract fails here.  The
kernels are held to the same checks in tests/test_frontend_fp64_gpu.py.

The bounds (oracle/frontend_cases.py; u = 2^-24):

* FPS distance.  d = ((dx*dx)+(dy*dy))+(dz*dz) with dx = fl(p - o): each difference carries a relative error u, each
  square 2u + u, the two additions u each, so |fl(d) - d64| <= 6u d64 (all terms are non-negative).  The running
  minimum is monotone, so the fp32 minimum keeps that bound against the float64 one.  The kernel's pick maximises the
  fp32 value, hence its float64 value lies within 12u vmax of the float64 maximum vmax; a step is decided when vmax
  beats the runner-up (the largest distinct value) by more than that margin, and a decided pick must be float64's
  arg-max.  Bitwise-equal points yield equal values, so any of the tied indices passes; the tie rule itself stays with
  test_fps_tie_rule_matches_block_reduction.  The skip mag = x*x+y*y+z*z <= 1e-3 (double literal) is decided outside
  4u 1e-3 of it (three products and two additions: <= 3u mag), and exactly when every fp32 partial sum is exact; a
  cloud where every point is skipped picks index 0 at every step.  idx[0] = 0 and kpts = xyz[idx] exactly.
* Radius histogram.  The reference's x^2 + y^2 - 2xy in fp32, in any order, FMA or not, is within c u (|k|^2 + |p|^2)
  of d64 = |k - p|^2: each norm and the dot product are within 3u of their magnitudes (3u (|k|^2 + |p|^2) for the
  norms, 3u |2 k.p| <= 3u (|k|^2 + |p|^2) for the doubled dot), the sum of the norms adds u (|k|^2 + |p|^2) and the
  final subtraction u |d|, with |d| <= 2 (|k|^2 + |p|^2) when p ~ -k: c = 3 + 3 + 1 + 2 = 9 to first order.  It is exact when every coordinate is a multiple of 2^-13 and (|k| + |p|)^2 < 1/4.  So for every
  m in 0..8192, #{d64 + e < thr_m} <= hist[m] <= #{d64 - e < thr_m}, thr_m = fl32(r_m^2).  The filter d2 <= 25 never
  changes a count (every thr_m <= 25).  pct = fl32(fl32(count) / fl32(N Kr)) * 100 is monotone in the count, so each
  bisection decision is decided when the pct of both ends lies on one side; the kernel's m must be reachable through
  the undecided ones, and equal when there are none.  Separately the reference loop is replayed literally (Python
  float64 bisection, torch fp32 percentage, round(des_r, 2)) on the kernel's own cumulative histogram: it must give the
  same m and float32(round(5 m / 8192, 2)), which pins the bisection exactly.
* Patch hits.  d2 as for FPS: within 6u d64, so a hit d64 < fl32(r * r) is decided outside 7u of it, and exactly when
  every fp32 intermediate is exact.  Each index row is strictly increasing over its listed prefix; every listed entry
  is a hit or undecided; no decided hit is skipped below the last listed entry; with fewer than P listed no decided hit
  is missing; the rest repeats the first index, and an empty ball gives all zeros.  Patches are copies, so they must
  equal the float64 mask formula applied to the row exactly.

Mutations of the oracle each of these tests catches are listed in DESIGN.md section 7."""
from ctypes import c_int64

import numpy as np
import pytest
import torch

from oracle import frontend_cases as F
from oracle.frontend_cases import merge, report


def _bisect_m(oracle, cum, denom, th, tol):
    return int(oracle.lib().bxo_radius_bisect(oracle._p(np.ascontiguousarray(cum, np.int64)), c_int64(denom), float(th), float(tol)))


# ------------------------------------------------------------------------------------------------ a1
@pytest.mark.parametrize("kind", F.FPS_KINDS)
@pytest.mark.parametrize("offset", [0.0, 1e3, 1e4])
def test_fps_oracle_vs_fp64(oracle, kind, offset):
    """npoint 1, N and more than the points left after the skip; N = 1."""
    acc = {}
    for n in (1, 37, 300):
        xyz = F.fps_cloud(kind, n, seed=n, offset=offset if kind not in ("allskip", "fewvalid", "magedge") else 0.0)
        for npoint in sorted({1, n, min(n + 5, 2 * n), 8}):
            merge(acc, F.check_fps(xyz, npoint, oracle.fps(xyz, npoint)))
    report(f"fps {kind} offset {offset:g}", acc)


def test_fps_skip_edges_are_exact(oracle):
    """The fp32 values either side of 1e-3: 1e-3f (just above; its points have exact magnitudes, so float64 decides
    them) is a candidate, its neighbour below is skipped; an fp32 compare against 1e-3f, or a swapped skip, changes
    the picks."""
    xyz = F.fps_cloud("magedge", 64, seed=3)
    mag = lambda p: ((p[0] * p[0]) + (p[1] * p[1])) + (p[2] * p[2])
    assert mag(xyz[64 // 3]) == F.MAG_HI and mag(xyz[0]) == F.MAG_LO
    n_lo = sum(mag(p) == F.MAG_LO for p in xyz)
    idx = oracle.fps(xyz, 64)
    assert oracle.fps_fp64(xyz, idx)["n_undecided_skip"] == n_lo
    mags = [mag(xyz[k]) for k in idx[1:]]
    assert F.MAG_HI in mags and F.MAG_LO not in mags
    merge({}, F.check_fps(xyz, 64, idx))


# ------------------------------------------------------------------------------------------------ a2
@pytest.mark.parametrize("kind", F.RADIUS_KINDS)
def test_radius_oracle_vs_fp64(oracle, kind):
    kp, pts = F.radius_case(kind, n=2500, kr=48, seed=len(kind))
    cum = oracle.radius_hist(kp, pts)
    lo, hi = oracle.radius_count_bounds(kp, pts)
    denom = len(pts) * len(kp)
    ths = F.RADIUS_THRESHOLDS
    radii = oracle.radius_estimation(pts[:1], kp, pts, kp, ths)
    ms = [_bisect_m(oracle, cum, denom, th, 0.01) for th in ths]
    out = F.check_radius(cum, denom, ths, 0.01, ms, radii, lo, hi)
    if kind == "axis":
        assert out["hist_undecided_bins"] == 0, "exact pairs must give exact counts"
    if kind == "dense":
        assert np.float32(radii[2]) == 0.0, "the dense cloud's 0.5 % radius rounds to 0.0"
    if kind == "far":
        assert cum[-1] == 0 and radii == [5.0, 5.0, 5.0]
    report(f"radius {kind}", out)


def test_radius_bisect_tolerance_edges(oracle):
    """pct exactly at threshold - tolerance and threshold + tolerance (25 % at the first probe, m = 4096): both are
    inside the band, so the loop stops there."""
    denom = 65536
    cum = 4 * np.arange(8193, dtype=np.int64)
    lo = hi = cum
    for th, tol in ((20.0, 5.0), (30.0, 5.0), (25.0, 0.0)):
        m = _bisect_m(oracle, cum, denom, th, tol)
        reach, und, radii = oracle.radius_fp64(lo, hi, denom, th, tol)
        assert reach == {4096} and und == 0 and m == 4096
        assert oracle.radius_replay(cum, denom, th, tol) == (4096, np.float32(2.5))


@pytest.mark.parametrize("ns,nt", [(1800, 1500), (1600, 1600), (1500, 1800)])
def test_radius_cloud_choice(oracle, ns, nt):
    """The source only when it has strictly more points; on a tie the target (a denser one here) wins."""
    kps, src = F.radius_case("uniform", n=ns, kr=32, seed=1)
    kpt, tgt = F.radius_case("dense", n=nt, kr=32, seed=2)
    ths = F.RADIUS_THRESHOLDS
    radii = oracle.radius_estimation(src, kps, tgt, kpt, ths)
    e = oracle.radius_estimation_fp64(src, kps, tgt, kpt, ths)
    for r, (reach, und, rad) in zip(radii, e["per"]):
        assert np.float32(r) in set(rad.values())
    other = oracle.radius_estimation(tgt, kpt, src, kps, ths)
    assert (radii != other) == (ns == nt)


def test_radius_subsampled_route(oracle):
    """Above 200000 points: pts[sub_idx] histogrammed, the denominator keeps the original N."""
    rng = np.random.default_rng(5)
    kp, pts = F.radius_case("uniform", n=300000, kr=6, seed=5)
    sub = rng.integers(0, len(pts), 200000)
    ths = F.RADIUS_THRESHOLDS
    radii = oracle.radius_estimation(pts[:10], kp[:6], pts, kp, ths, sub_idx=sub)
    e = oracle.radius_estimation_fp64(pts[:10], kp[:6], pts, kp, ths, sub_idx=sub)
    assert e["denom"] == 300000 * 6
    cum = oracle.radius_hist(kp, pts[sub])
    ms = [_bisect_m(oracle, cum, e["denom"], th, 0.01) for th in ths]
    report("radius 300000 points sub-sampled", F.check_radius(cum, e["denom"], ths, 0.01, ms, radii, e["lo"], e["hi"]))


# ------------------------------------------------------------------------------------------------ a3
@pytest.mark.parametrize("kind", F.PATCH_KINDS)
@pytest.mark.parametrize("offset,r", [(0.0, None), (1e3, 0.1), (1e4, 0.05)])
def test_patches_oracle_vs_fp64(oracle, kind, offset, r):
    acc = {}
    P = 16
    pts, kp, rr = F.patch_case(kind, n=2000, k=48, r=r or 0.3, P=P, seed=3, offset=offset)
    rng = np.random.default_rng(1)
    perm = rng.permutation(len(pts)).astype(np.int32)
    for radius in (rr, 0.0):
        idx, patches = oracle.select_patches(pts, perm, kp, radius, P)
        merge(acc, F.check_ball_query(pts[perm], kp, radius, idx))
        merge(acc, F.check_patches(pts[perm], kp, idx, patches))
        bidx, _ = oracle.ball_query(pts[perm], kp, radius, P)
        assert np.array_equal(bidx, idx)
    if kind == "counts":
        assert acc["bq_full"] >= 2 * (48 // 3)
    if kind == "exact":
        assert acc["bq_undecided_listed"] < acc["bq_rows"] * P
    report(f"patches {kind} offset {offset:g}", acc)
