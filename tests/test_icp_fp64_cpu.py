"""The float64 ICP oracle (oracle/icp_fp64.py) on cases with a known answer, the grid window of csrc/bx_icp.cu, and the
oracle mutations these checks catch.  No GPU.

Bounds used by tests/test_icp_gpu.py (oracle/icp_cases.py), with u53 = 2^-53:
- Points.  The GPU's transformed source after k updates differs from the oracle's by at most
      delta_k = |dR_k|_F X + |dt_k| + 2 (k + 1) KD u53 (X + |t|),   X = sqrt(3) max |src|,
  where dR_k, dt_k are the measured differences of the two transformations: both sides apply the same rigid maps up to
  dR_k, dt_k, and each incremental application rounds a coordinate ((u0 x + u1 y) + u2 z) + u3 by at most 4 roundings of
  terms below |p| + |t| (KD = 16 covers them with a factor 4).
- Decisions.  Moving a point by delta changes its d2 = |q - p|^2 by at most (2r + delta) delta for every target within
  reach, so a point's decision is fixed when |d2_nearest - r^2| > D and the gap to the second-nearest target > 2D,
  D = 2 (2r + delta) delta + 8 u53 r^2 (a factor 2 and the rounding of d2).  A step with no point inside those margins is
  decided: its correspondence set must equal the oracle's and so must its fitness.  At an undecided step with m marginal
  points, at most m correspondences may differ and fitness may move by m / N.
- rmse.  With equal correspondences, |d rmse| <= delta_k (rmse is an l2 mean of distances, each moved by <= delta_k) plus
  the rounding of the sums, KS (n + 16) u53 max(rmse, r) (KS = 64: the sums are blocked, no term exceeds r^2).  With m
  marginal points it may move by r sqrt(2 m / (n_corr - m)) more (each flipped point contributes at most r^2 to a sum).
- Transformation.  One Umeyama solve on the same correspondences differs by rounding only: the moments by a few u53 of
  their magnitude (taken about a point near the data), and the polar factor R of Sigma by at most 2 |dSigma| / (s2 + s3),
  i.e. |dR|_F <= KT u53 (1 + kappa), kappa = s1 / (s2 + s3), KT = 2^12.  The final bound sums that over the steps (an
  upper bound: ICP contracts earlier errors) and takes |dt| <= the same times (|centroid| + 1 + |t|).  Where the fit is
  not unique (a planar target's rotation about its normal, one or two correspondences) the residuals are held instead.
"""
import math

import numpy as np
import pytest

from oracle import icp_cases as C
from oracle.icp_fp64 import icp_fp64, xform

F32 = np.float32


def run(name, mutations=(), **kw):
    c = C.case(name)
    args = dict(init=c["init"], max_iteration=c["max_iteration"])
    args.update(kw)
    return c, icp_fp64(c["src"], c["tgt"], c["r"], _mutations=mutations, **args)


def check_known_transform(name, mutations=()):
    c, out = run(name, mutations)
    T = c["T_true"]
    scale = 1.0 + float(np.abs(T[:3, 3]).max()) + float(np.abs(c["tgt"]).max())
    assert np.abs(out["T"][:3, :3] - T[:3, :3]).max() < 1e-10, out["T"] - T
    assert np.abs(out["T"][:3, 3] - T[:3, 3]).max() < 1e-10 * scale, out["T"] - T
    assert out["fitness"] == 1.0 and out["rmse"] < 1e-10 * scale and out["converged"]
    return out


@pytest.mark.parametrize("name", ["exact", "init", "offset"])
def test_known_rigid_motion(name):
    """Noise-free full overlap: the oracle ends on the motion the clouds were made with (also from a non-identity init and
    1e4 m from the origin), with fitness 1 and rmse 0."""
    out = check_known_transform(name)
    assert out["iterations"] >= 2


def test_max_iteration_0_and_1():
    c, out0 = run("init", max_iteration=0)
    assert out0["iterations"] == 0 and np.array_equal(out0["T"], c["init"]) and len(out0["steps"]) == 1
    _, out1 = run("init", max_iteration=1)
    assert out1["iterations"] == 1 and np.array_equal(out1["T"], out1["steps"][1]["update"] @ c["init"])
    _, full = run("init")
    assert np.array_equal(full["steps"][1]["T"], out1["T"]) and full["steps"][1]["fitness"] == out1["fitness"]


def test_no_correspondences():
    """Clouds 10 m apart: identity, fitness 0, rmse 0, and the loop stops after one step (nothing changed)."""
    c, out = run("none")
    assert np.array_equal(out["T"], np.eye(4)) and out["fitness"] == 0.0 and out["rmse"] == 0.0
    assert out["iterations"] == 1 and out["converged"] and (out["corr"] < 0).all()


def check_points_at_r(mutations=()):
    """d2 exactly r*r (dyadic points, exact in float64) is not a correspondence; 0.25 m away is."""
    c, out = run("at_r", mutations)
    corr = out["steps"][0]["corr"]
    assert list(corr) == [-1, -1, -1, 3], corr


def test_points_at_r():
    check_points_at_r()


def check_incremental(name, mutations=()):
    """pcd is the source moved by init and then by every update in turn, each application in the fixed order -- bit for bit;
    it is not the source moved once by the accumulated transformation."""
    c, out = run(name, mutations)
    p = c["src"].copy() if np.array_equal(c["init"], np.eye(4)) else xform(c["init"], c["src"])
    for st in out["steps"][1:]:
        p = xform(st["update"], p)
    assert np.array_equal(p, out["pcd"])
    return out


@pytest.mark.parametrize("name", ["exact", "init", "offset"])
def test_pcd_is_transformed_incrementally(name):
    out = check_incremental(name)
    c = C.case(name)
    once = xform(out["T"], c["src"])
    assert not np.array_equal(once, out["pcd"])          # the two orders round differently on these clouds


def check_proper_rotation(name, mutations=()):
    """Every update is a rotation (det +1, orthonormal) -- also where the best orthogonal map is a reflection (mirror) and
    where the target is scaled (scaled)."""
    c, out = run(name, mutations)
    for st in out["steps"][1:]:
        R = st["update"][:3, :3]
        assert np.abs(R.T @ R - np.eye(3)).max() < 1e-12 and np.linalg.det(R) > 0, R


@pytest.mark.parametrize("name", ["mirror", "scaled", "exact"])
def test_updates_are_rotations(name):
    check_proper_rotation(name)


def test_ties_take_the_lowest_index():
    c, out = run("dup")
    n = c["tgt"].shape[0] // 2
    st = out["steps"][0]
    assert (st["corr"][st["corr"] >= 0] < n).all()   # t[i] is at i and 2n - 1 - i; the lower index always wins
    assert (st["margin_gap"][st["corr"] >= 0] == 0.0).all()


def test_refusals():
    c = C.case("exact")
    with pytest.raises(ValueError):
        icp_fp64(c["src"], c["tgt"], 0.0)
    with pytest.raises(ValueError):
        icp_fp64(c["src"], c["tgt"], -1.0)
    with pytest.raises(ValueError):
        icp_fp64(np.zeros((0, 3)), c["tgt"], 0.5)


# the test that notices each oracle mutation
MUTATIONS = [
    ("le", lambda m: check_points_at_r(m)),
    ("retransform", lambda m: check_incremental("init", m)),
    ("right_mul", lambda m: check_known_transform("init", m)),
    ("no_det_fix", lambda m: check_proper_rotation("mirror", m)),
    ("with_scaling", lambda m: check_proper_rotation("scaled", m)),
    ("fitness_only", lambda m: check_known_transform("exact", m)),
    ("origin_moments", lambda m: check_known_transform("offset", m)),
]


@pytest.mark.parametrize("mutation,check", MUTATIONS, ids=[m for m, _ in MUTATIONS])
def test_mutation_is_caught(mutation, check):
    check(())                                            # passes on the oracle as written
    with pytest.raises(AssertionError):
        check((mutation,))


# --------------------------------------------------------------------------------------------------------------------
# grid window of csrc/bx_icp.cu (icp_window), in fp32 with the kernel's arithmetic
def _rf(r):
    rf = F32(r)
    return np.nextafter(rf, F32(np.inf)) if float(rf) < r else rf


def _ic(r):
    return F32(1.0) / (_rf(r) * F32(1.001))


def _window(a):
    a = np.asarray(a, F32)
    w = (F32(0.9993) + (F32(2.0 ** -21) * np.abs(a)).astype(F32)).astype(F32)
    return np.floor((a - w).astype(F32)).astype(np.int64), np.floor((a + w).astype(F32)).astype(np.int64)


def _pairs(r, centre, extent, n, seed):
    """float64 queries and targets just inside r (random and axis directions), as the kernel sees them."""
    rng = np.random.default_rng(seed)
    q = centre + rng.uniform(-extent, extent, size=(n, 3))
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    d[: n // 2] = np.eye(3)[rng.integers(0, 3, n // 2)] * rng.choice([-1.0, 1.0], size=(n // 2, 1))
    p = q + d * rng.uniform(0.99, 1.0, size=(n, 1)) * r
    return q, p


def _check_window(q, p, r):
    from oracle.icp_fp64 import d2_fixed
    hit = d2_fixed(q, p) < r * r
    ic = _ic(r)
    a = (q.astype(F32) * ic).astype(F32)
    b = (p.astype(F32) * ic).astype(F32)
    lo, hi = _window(a)
    cell = np.floor(b).astype(np.int64)
    inside = (cell >= lo) & (cell <= hi)
    ok = (np.abs(a) < 2.0 ** 19).all(1)
    assert inside.all(1)[hit & ok].all(), "a hit outside the query window"
    return hit, hi - lo + 1, a, ok


@pytest.mark.parametrize("r,centre,extent", [(0.2, 0.0, 80.0), (0.2, 1e4, 50.0), (0.05, 2.5e4, 10.0), (0.2, -1e4, 50.0),
                                             (0.1, 0.0, 5.0), (1.7, 3e5, 100.0), (0.2, 1.0e5, 50.0)])
def test_window_encloses_every_hit(r, centre, extent):
    """Large coordinates included: 1e4 m (5e4 cells at r = 0.2) up to 1e5 m (2^19 cells, where the kernel still uses it)."""
    q, p = _pairs(r, centre, extent, 400000, int(r * 100) + int(abs(centre)) % 1000)
    hit, n, a, ok = _check_window(q, p, r)
    assert hit.mean() > 0.9 and ok.mean() > 0.99
    assert n[ok].max() <= 4 and (n[(np.abs(a) < 1468).all(1)] <= 3).all()


@pytest.mark.parametrize("k", [12, 14, 16, 17, 18])
def test_window_across_power_of_two_cells(k):
    """Queries whose cell values straddle 2^k, where fp32 cell coordinates jump."""
    r = 0.2
    centre = 2.0 ** k / float(_ic(r))
    q, p = _pairs(r, centre, 4 * r, 200000, k)
    _check_window(q, p, r)
    _check_window(-q, -p, r)


def test_window_sizes():
    """3 cells per axis below ~1468 cells from the origin (27 buckets), at most 4 below 2^19 (64 buckets)."""
    a = np.concatenate([np.linspace(-1468, 1468, 2_000_001), np.linspace(-2.0 ** 19 + 1, 2.0 ** 19 - 1, 2_000_001)]).astype(F32)
    lo, hi = _window(a)
    n = hi - lo + 1
    assert (n[: 2_000_001] <= 3).all() and (n <= 4).all() and (n >= 2).all()
    assert math.isclose(float(_rf(0.2)), 0.2, rel_tol=1e-7) and float(_rf(0.2)) >= 0.2


@pytest.mark.parametrize("bias", [1.01, 1.001, 1.0 + 1e-7])
@pytest.mark.parametrize("name", ["exact", "offset", "kitti"])
def test_step_check_refuses_a_biased_transformation(monkeypatch, name, bias):
    """The GPU-side step check holds the transformation to an a-priori bound before it uses the measured difference: a
    run whose every Umeyama translation is scaled by `bias` fails at the first update, however small the bias (a check that
    widened its tolerances with the measured error would pass it)."""
    import oracle.icp_fp64 as O
    c = C.kitti_pair(0, n=8000) if name == "kitti" else C.case(name)
    out = icp_fp64(c["src"], c["tgt"], c["r"], init=c["init"], max_iteration=c["max_iteration"])
    exact = icp_fp64(c["src"], c["tgt"], c["r"], init=c["init"], max_iteration=1)
    g = dict(T=exact["T"], fitness=exact["fitness"], rmse=exact["rmse"], corr=exact["corr"])
    assert C.check_step(g, out, 1, c["src"], c["r"], c["hold"])[0]          # the unbiased run passes, decided
    umeyama = O.umeyama

    def biased(s, t, mutations=()):
        T, D = umeyama(s, t, mutations)
        T = T.copy()
        T[:3, 3] *= bias
        return T, D

    monkeypatch.setattr(O, "umeyama", biased)
    b = icp_fp64(c["src"], c["tgt"], c["r"], init=c["init"], max_iteration=1)
    with pytest.raises(AssertionError, match="T differs"):
        C.check_step(dict(T=b["T"], fitness=b["fitness"], rmse=b["rmse"], corr=b["corr"]), out, 1, c["src"], c["r"], c["hold"])
