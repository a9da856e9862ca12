"""The loader bootstrap (f1) and the cpp_wrappers ports (a17, a18) against float64, sklearn and the reference's own C++,
without a GPU.  The oracle's pca_alignment, sphericity_based_voxel_analysis, voxel_down_sample, radius_neighbors and
grid_subsample are held to the checks of oracle/bootstrap_cases.py; the kernels are held to the same checks in
tests/test_bootstrap_fp64_gpu.py.  The references are numpy's eigh of the centred 1/(n-1) covariance, sklearn's
PCA(n_components=3) itself, np.unique over float64 voxel tuples, and the reference's compiled cpp_wrappers
(tests/golden/reference_cpp_edges.npz, written by tests/tools/gen_reference_cpp_edges.py).

The bounds (u = 2^-53 for float64 work, u24 = 2^-24 for fp32 work):

* Mean.  n fp32 points summed in float64 in any order, then divided: |dm| <= (n + 1) u mean|x| (the kernel's atomics
  and numpy's pairwise sum each), checked at twice that.
* Covariance and eigenvalues.  The kernel centres on its own mean m + dm: sum (x - m - dm)(y - m' - dm') = sum dx dy +
  n dm dm' (the first-order terms vanish because sum dx = 0), each difference and product adds u |dx dy|, the sum
  (n - 1) u sum |dx dy|: E_ab = ((n + 6) u sum |dx_a||dx_b| + n |dm_a dm_b|) / (n - 1).  By Weyl every eigenvalue moves
  by at most ||E||_2 <= ||E||_F; the 3x3 cyclic Jacobi (or LAPACK, or sklearn's SVD) adds a backward error of a few u
  ||C||, taken as 64 u ||C||_F per side: e_lam = 2 ||E||_F + 128 u ||C||_F for two evaluations.
* Components.  Davis-Kahan: sin(angle) <= e_lam / gap, gap = the distance of the row's eigenvalue to the others;
  ||v - v'|| = 2 sin(angle / 2) <= 1.5 e_lam / gap = e_v.  A row is checked where e_v < 0.1 (the gap determines it);
  the rod's, disc's and ball's degenerate rows are counted instead.  Its sign is checked where the two largest
  |entries| differ by more than 2 e_v (otherwise the sign rule may legitimately choose either); the returned row must
  still satisfy the rule (largest |entry| positive, first index on a tie).
* z-range.  With the kernel's own mean and axis every projection is within 4 u sum_c |p_c - m_c||a_c| of the exact
  value (one difference, one product, two sums per term); two evaluations: 10 u max_i sum_c |p_ic - m_c||a_c|.  Against
  the reference's range the axis itself moves: 2 sqrt3 max|p - m| (2 e_v) more, plus 36 u max|p|.
* Decisions.  sphericity = l3 / l1 moves by e_lam (1 + sph) / l1; |z . e_z| by e_v; z_s . z_t by e_v(s) + e_v(t) and only
  where both signs are decided; voxel = sqrt(z_range) / 100 alpha by alpha e_zr / (200 sqrt(z_range)).  Each of
  (round(voxel, 4), sphericity, is_aligned) must equal sklearn's where its float64 margin exceeds its bound (alpha needs
  the sphericity decision, the flag is three-valued: one decided False decides it); the rest are listed with margins.
* Voxel down-sampling.  index = floor((p - (min - voxel / 2)) / voxel) is evaluated in float64 on the fp32 points by
  the kernel and by Open3D alike, so the voxel set is exact: it is compared as (ix, iy, iz) tuples of np.unique(axis=0),
  not as the oracle's masked key.  Means: fp64 sums in any order, then one fp32 rounding: u24 |mean| + (cnt + 2) u
  max|p|.  The loader's second call gets the kernel's fp32 means where Open3D keeps doubles: they differ by that bound
  dm, the second grid's origin by max dm, so a first-stage voxel may land in another second-stage cell only within
  (dm + max dm) / voxel0 of a cell boundary (1 % slack, plus 4 u of the index).  float64 input is rounded to fp32 by
  bootstrap._cloud: the same rule with dm = |p - fl32(p)|.  A cloud spanning 2^21 voxels or more on an axis is refused:
  the key holds 21 bits per axis.
* Barycentres (a18).  fp32 sums in any order, fl32(1 / cnt) and the product: (cnt + 2) u24 (max|b| + 2 dl) per
  coordinate, twice for two summation orders.  Keys and counts are exact; the oracle's barycentres equal the
  reference's bit for bit (both sum in input order).
* Neighbours (a17).  d = ((dx dx) + (dy dy)) + (dz dz) in float64 from fp32 coordinates is exact up to the reference's own
  rounding, which the kernel repeats: distance sequences must be equal, every entry d < fl32(r * r) and no other
  support of the searched cloud.  nanoflann sorts with std::sort, which is not stable: inside a run of equal distance
  only the index set is compared with the reference; the oracle's and the kernel's order is (distance, index).

The largest ratios (error / bound) are printed with -s and recorded in DESIGN.md section 7."""

import numpy as np
import pytest

from oracle import bootstrap_cases as B
from oracle.bootstrap_cases import merge, report

EDGES = B.load_edges()


# ------------------------------------------------------------------------------------------------ f1: PCA
@pytest.mark.parametrize("kind", B.PCA_KINDS)
def test_pca_oracle_and_sklearn_vs_fp64(oracle, kind):
    acc = {}
    for seed in (0, 1):
        pts, idx = B.pca_cloud(kind, seed=seed)
        sph, aligned, mean, var, comps = oracle.pca_alignment(pts, idx)
        merge(acc, B.check_pca(pts, idx, mean, var, comps))
        merge(acc, {"sklearn_" + k: v for k, v in B.check_sklearn(pts, idx).items()})
    if kind in ("generic", "plane", "offset1e5", "offset5e5", "mm"):
        assert acc["n_comp_undetermined"] == 0
    expect = {"rod": 8, "disc": 8, "ball": 12}                          # degenerate rows x two seeds x (oracle, sklearn)
    assert acc["n_comp_undetermined"] + acc["sklearn_n_comp_undetermined"] == expect.get(kind, 0)
    if kind == "rot45":
        assert acc["n_sign_undecided"] == 4           # rows (1, 1, 0) and (1, -1, 0) tie under the sign rule, two seeds
    report(f"pca {kind}", acc)


def test_pca_refuses_fewer_than_three_samples(oracle):
    """A 29-point cloud samples int(29 / 10) = 2 points: sklearn refuses, so does the oracle; 30 points (3 samples)
    pass."""
    from sklearn.decomposition import PCA
    pts = B.pca_cloud("n30", seed=3)[0].astype(np.float64)
    idx2 = B.sample(29, 3)
    assert len(idx2) == 2
    with pytest.raises(ValueError):
        PCA(n_components=3).fit(pts[idx2])
    with pytest.raises(ValueError, match="n_components=3"):
        oracle.pca_alignment(pts[:29], idx2)
    idx3 = B.sample(30, 3)
    merge({}, B.check_pca(pts, idx3, *oracle.pca_alignment(pts, idx3)[2:]))


def test_analysis_oracle_vs_sklearn(oracle):
    acc, undecided = {}, []
    for name, s, t, i_s, i_t in B.analysis_pairs():
        rf = B.reference_analysis(s, t, i_s, i_t)
        out = B.check_analysis(oracle.sphericity_based_voxel_analysis(s, t, i_s, i_t), rf)
        undecided += [(name,) + u for u in out.pop("undecided")]
        if name.split()[-1] in ("-1e-03", "+1e-03", "-1e-06", "+1e-06"):
            assert out["n_undecided"] == 0, name
        merge(acc, out)
    report("analysis", acc)
    print("undecided (decision, float64 margin, bound):", undecided)


# ------------------------------------------------------------------------------------------------ f1: voxel down-sampling
@pytest.mark.parametrize("kind", B.VDS_KINDS)
def test_voxel_down_sample_oracle_vs_fp64(oracle, kind):
    acc = {}
    for seed in (0, 1):
        pts, voxel = B.vds_cloud(kind, seed)
        keys, means, cnt = oracle.voxel_down_sample(pts, voxel)
        merge(acc, B.check_vds(pts, voxel, keys, means.astype(np.float32), cnt))
    report(f"voxel_down_sample {kind}", acc)


@pytest.mark.parametrize("voxel", [0.05, 0.001])
def test_voxel_down_sample_refuses_2_21_cells(oracle, voxel):
    """Before, two points 104 857.6 m apart at voxel 0.05 became one voxel at their midpoint (the key masks 21 bits per
    axis); the oracle now refuses an axis of 2^21 voxels, and keeps the two voxels just inside it."""
    inside, beyond = B.axis_limit_cloud(voxel)
    keys, means, cnt = oracle.voxel_down_sample(inside, voxel)
    assert len(keys) == 2
    merge({}, B.check_vds(inside, voxel, keys, means, cnt))
    with pytest.raises(ValueError, match="2\\^21"):
        oracle.voxel_down_sample(beyond, voxel)
    far = np.array([[0, 0, 0], [0, 104857.6, 0]], np.float32)
    with pytest.raises(ValueError, match="2\\^21"):
        oracle.voxel_down_sample(far, 0.05)


def test_voxel_down_sample_refuses_non_finite(oracle):
    with pytest.raises(ValueError, match="finite"):
        oracle.voxel_down_sample(np.array([[0, 0, 0], [np.inf, 1, 1]], np.float32), 0.05)


def test_loader_route_oracle(oracle):
    """The check of the loader's two calls, fed the oracle's means rounded to fp32 (what the kernel returns)."""
    acc = {}
    for name, pts, ds in B.loader_clouds():
        k1, m1, c1 = oracle.voxel_down_sample(pts, ds)
        for voxel0 in (0.035, 0.30):
            x1 = m1.astype(np.float32)
            k2, m2, c2 = oracle.voxel_down_sample(x1, voxel0)
            merge(acc, B.check_loader_route(pts, ds, voxel0, (k1, x1, c1), (k2, m2.astype(np.float32), c2)))
    report("loader route (oracle)", acc)


def test_fp64_input_oracle(oracle):
    P64 = B.pca_cloud("generic", 20000, 7)[0].astype(np.float64) + np.random.default_rng(7).normal(scale=1e-6, size=(20000, 3))
    acc = {}
    for voxel in (0.035, 0.3):
        k, m, c = oracle.voxel_down_sample(P64.astype(np.float32), voxel)
        merge(acc, B.check_fp64_input(P64, voxel, k, m.astype(np.float32), c))
    report("float64 input (oracle)", acc)


# ------------------------------------------------------------------------------------------------ a17 / a18 against the C++
def test_edges_golden_inputs_are_the_cases():
    for name, (q, s, qb, sb, r) in B.neighbor_cases().items():
        assert np.array_equal(EDGES[f"nb_{name}_q"], q) and np.array_equal(EDGES[f"nb_{name}_s"], s), name
    for name, (p, dl) in B.subsample_cases().items():
        assert np.array_equal(EDGES[f"gs_{name}_p"], p), name


def test_edges_golden_equals_the_compiled_reference(oracle):
    if not oracle.ref_available():
        pytest.skip("oracle/_ref/libbxref.so is built only where the reference checkout is present")
    for name, (q, s, qb, sb, r) in B.neighbor_cases().items():
        got = oracle.ref_radius_neighbors(q, s, qb, sb, r)
        ref = EDGES[f"nb_{name}_ref"]
        assert got.shape == ref.shape, name
        merge({}, B.check_neighbors(q, s, qb, sb, r, oracle.radius_neighbors(q, s, qb, sb, r), ref=got))
    for name, (p, dl) in B.subsample_cases().items():
        assert np.array_equal(B._bitsort(oracle.ref_grid_subsampling(p, dl)), B._bitsort(EDGES[f"gs_{name}_ref"])), name


@pytest.mark.parametrize("name", list(B.neighbor_cases()))
def test_radius_neighbors_oracle_vs_reference_edges(oracle, name):
    q, s, qb, sb, r = B.neighbor_cases()[name]
    ref = EDGES[f"nb_{name}_ref"]
    got = oracle.radius_neighbors(q, s, qb, sb, r)
    out = B.check_neighbors(q, s, qb, sb, r, got, ref=ref)
    if name == "empty":
        assert got.shape == (len(q), 0)
    if name == "ball4096":
        assert got.shape[1] > 4096
    if name == "sqrt5":                       # points at d^2 = 5 = fl32(r * r) are excluded, float64's r^2 would keep them
        d = B.row_distances(q[0], s, np.arange(len(s)))
        assert (d == 5.0).any() and (d < float(B.R_SQRT5) ** 2).sum() > (d < 5.0).sum()
    report(f"radius_neighbors {name}", out)


def grid_keys_np(p, dl, wrap=True):
    """a18's cell keys evaluated in fp32 numpy: wrap=True casts the cell index through int64 (the reference's x86 build,
    the oracle, the kernel); wrap=False clamps it at 0 (a direct float -> u64 conversion on the GPU)."""
    p = np.asarray(p, np.float32)
    dl = np.float32(dl)
    inv = np.float32(1) / dl
    org = (np.floor(p.min(0) * inv) * dl).astype(np.float32)
    cast = (lambda v: v.astype(np.int64).astype(np.uint64)) if wrap else (lambda v: np.maximum(v, 0).astype(np.uint64))
    NX, NY = cast(np.floor((p.max(0)[:2] - org[:2]) / dl)) + np.uint64(1)
    i = cast(np.floor((p - org) / dl))
    with np.errstate(over="ignore"):
        return i[:, 0] + NX * i[:, 1] + NX * NY * i[:, 2]


@pytest.mark.parametrize("name", list(B.subsample_cases()))
def test_grid_subsample_oracle_vs_reference_edges(oracle, name):
    p, dl = B.subsample_cases()[name]
    ref = EDGES[f"gs_{name}_ref"]
    keys, xyz, cnt = oracle.grid_subsample(p, dl)
    out = B.check_subsample(p, dl, keys, xyz, cnt, ref, (keys, xyz, cnt))
    assert np.array_equal(np.unique(grid_keys_np(p, dl)), keys)
    if name.startswith("above"):
        # the minimum corner gets cell -1: its key wraps to 2^64 - 1, the edge points alias onto the far row; a clamping
        # cast gives other cells than the reference
        assert keys[-1] == np.uint64(2 ** 64 - 1) and out["n_wrapped"] >= 1
        assert len(np.unique(grid_keys_np(p, dl, wrap=False))) != len(ref) or \
            not np.array_equal(np.unique(grid_keys_np(p, dl, wrap=False)), keys)
    if name in ("flat_x", "pair_y"):
        # NX = 0 and every cell index on x is -1: the reference keeps one cell, key 2^64 - 1; clamping keeps many
        assert len(keys) == len(ref) == 1 and keys[0] == np.uint64(2 ** 64 - 1)
        assert len(np.unique(grid_keys_np(p, dl, wrap=False))) > 1
    if name == "flat_y":
        # NY = 0: the key ix + NX * iy forgets z, so fewer cells than (x, z) pairs occupied; clamping keeps them apart
        assert len(keys) == len(ref) and len(np.unique(grid_keys_np(p, dl, wrap=False))) > len(keys)
    report(f"grid_subsample {name}", out)
