"""The loader bootstrap kernels (bx_pca_analysis, bx_project_range, bx_voxel_down_sample) and the cpp_wrappers ports
(bx_radius_neighbors, bx_grid_subsample) on the edge inputs of oracle/bootstrap_cases.py, held to float64, sklearn and
the reference's own C++ (tests/golden/reference_cpp_edges.npz) under the bounds derived in
tests/test_bootstrap_fp64_cpu.py.  Largest ratios print with -s."""
import numpy as np
import pytest
import torch

from oracle import bootstrap_cases as B
from oracle.bootstrap_cases import merge, report

pytestmark = pytest.mark.gpu

EDGES = B.load_edges()


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda", torch.cuda.current_device())


def cu(a, dev, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device=dev, dtype=dtype)


# ------------------------------------------------------------------------------------------------ f1: PCA and z-range
@pytest.mark.parametrize("kind", B.PCA_KINDS)
def test_pca_and_range_vs_fp64(dev, kind):
    from bufferx_b200 import ops
    acc = {}
    for seed in (0, 1):
        pts, idx = B.pca_cloud(kind, seed=seed)
        P = cu(pts, dev)
        mean, var, comps = ops.pca_analysis(P, cu(idx, dev, torch.int32))
        mean, var, comps = mean.cpu().numpy(), var.cpu().numpy(), comps.cpu().numpy()
        merge(acc, B.check_pca(pts, idx, mean, var, comps))
        for r in range(3):
            lo, hi = ops.project_range(P, cu(mean, dev, torch.float64), cu(comps[r], dev, torch.float64)).cpu().tolist()
            merge(acc, B.check_range(pts, mean, comps[r], lo, hi))
    expect = {"rod": 4, "disc": 4, "ball": 6}
    assert acc["n_comp_undetermined"] == expect.get(kind, 0)
    if kind == "rot45":
        assert acc["n_sign_undecided"] == 4
    report(f"pca {kind}", acc)


def test_project_range_multi_block(dev):
    """1 600 000 points: 592 blocks of 256 threads, each folding into the two ordered-integer atomics."""
    from bufferx_b200 import ops
    rng = np.random.default_rng(5)
    pts = (rng.normal(size=(1_600_000, 3)) * [20.0, 10.0, 2.0] + [300.0, -50.0, 4.0]).astype(np.float32)
    mean = pts[::7].astype(np.float64).mean(0)
    axis = np.array([0.1, -0.2, 0.97])
    axis /= np.linalg.norm(axis)
    lo, hi = ops.project_range(cu(pts, dev), cu(mean, dev, torch.float64), cu(axis, dev, torch.float64)).cpu().tolist()
    out = B.check_range(pts, mean, axis, lo, hi)
    report("project_range 1.6M", out)


def test_pca_refuses_fewer_than_three_samples(dev):
    from bufferx_b200 import ops
    from bufferx_b200.bootstrap import compute_pca_alignment
    from bufferx_b200.ops import BufferXError
    pts = cu(B.pca_cloud("n30", seed=3)[0], dev)
    with pytest.raises(ValueError, match="n_components=3"):
        compute_pca_alignment(pts[:29])                                  # int(29 / 10) = 2 samples, as sklearn refuses
    with pytest.raises(BufferXError, match="three samples"):
        ops.pca_analysis(pts, cu(np.array([0, 1]), dev, torch.int32))
    idx = B.sample(30, 3)
    mean, var, comps = compute_pca_alignment(pts, idx)[2]
    merge({}, B.check_pca(pts.cpu().numpy(), idx, mean.cpu().numpy(), var.cpu().numpy(), comps.cpu().numpy()))


def test_analysis_vs_sklearn(dev):
    from bufferx_b200.bootstrap import sphericity_based_voxel_analysis
    acc, undecided = {}, []
    for name, s, t, i_s, i_t in B.analysis_pairs():
        rf = B.reference_analysis(s, t, i_s, i_t)
        out = B.check_analysis(sphericity_based_voxel_analysis(s, t, i_s, i_t, device=dev), rf)
        undecided += [(name,) + u for u in out.pop("undecided")]
        merge(acc, out)
    report("analysis", acc)
    print("undecided (decision, float64 margin, bound):", undecided)


# ------------------------------------------------------------------------------------------------ f1: voxel down-sampling
@pytest.mark.parametrize("kind", B.VDS_KINDS)
def test_voxel_down_sample_vs_fp64(dev, kind):
    from bufferx_b200 import ops
    acc = {}
    for seed in (0, 1):
        pts, voxel = B.vds_cloud(kind, seed)
        keys, xyz, cnt = ops.voxel_down_sample(cu(pts, dev), voxel)
        merge(acc, B.check_vds(pts, voxel, keys.cpu().numpy(), xyz.cpu().numpy(), cnt.cpu().numpy()))
    report(f"voxel_down_sample {kind}", acc)


@pytest.mark.parametrize("voxel", [0.05, 0.001])
def test_voxel_down_sample_refuses_2_21_cells(dev, voxel):
    from bufferx_b200 import ops
    from bufferx_b200.ops import BufferXError
    inside, beyond = B.axis_limit_cloud(voxel)
    keys, xyz, cnt = ops.voxel_down_sample(cu(inside, dev), voxel)
    merge({}, B.check_vds(inside, voxel, keys.cpu().numpy(), xyz.cpu().numpy(), cnt.cpu().numpy()))
    for cloud in (beyond, beyond[:, [1, 0, 2]], beyond[:, [2, 1, 0]]):       # each axis
        with pytest.raises(BufferXError, match="2\\^21"):
            ops.voxel_down_sample(cu(cloud, dev), voxel)
    with pytest.raises(BufferXError, match="2\\^21"):
        ops.voxel_down_sample(cu(np.array([[0, 0, 0], [0, 104857.6, 0]], np.float32), dev), 0.05)


def test_voxel_down_sample_refuses_non_finite_extent(dev):
    """An infinite coordinate, or an axis whose every coordinate is NaN, leaves no voxel grid: refused by name."""
    from bufferx_b200 import ops
    from bufferx_b200.ops import BufferXError
    for bad in ([[0, 0, 0], [np.inf, 1, 1]], [[0, np.nan, 0], [1, np.nan, 1]], [[0, 0, -np.inf], [1, 1, 1]]):
        with pytest.raises(BufferXError, match="finite"):
            ops.voxel_down_sample(cu(np.array(bad, np.float32), dev), 0.05)


def test_loader_route(dev):
    """voxel_down_sample(downsample) then voxel_down_sample(voxel_size_0) on its fp32 output, against the float64
    chain, for the downsample the kernel's own analysis gives (the same as sklearn's on these clouds)."""
    from bufferx_b200 import ops
    from bufferx_b200.bootstrap import sphericity_based_voxel_analysis
    acc = {}
    for name, pts, ds in B.loader_clouds():
        n = len(pts)
        got = sphericity_based_voxel_analysis(pts, pts, B.sample(n, 0 if name == "generic" else 1),
                                              B.sample(n, 1 if name == "generic" else 2), device=dev)
        assert got[0] == ds, (got, ds)
        first = [a.cpu().numpy() for a in ops.voxel_down_sample(cu(pts, dev), ds)]
        for voxel0 in (0.035, 0.30):
            second = [a.cpu().numpy() for a in ops.voxel_down_sample(cu(first[1], dev), voxel0)]
            merge(acc, B.check_loader_route(pts, ds, voxel0, first, second))
    report("loader route", acc)


def test_fp64_input(dev):
    from bufferx_b200 import ops
    from bufferx_b200.bootstrap import _cloud, voxel_down_sample
    P64 = B.pca_cloud("generic", 20000, 7)[0].astype(np.float64) + np.random.default_rng(7).normal(scale=1e-6, size=(20000, 3))
    acc = {}
    for voxel in (0.035, 0.3):
        keys, xyz, cnt = ops.voxel_down_sample(_cloud(P64, dev), voxel)
        merge(acc, B.check_fp64_input(P64, voxel, keys.cpu().numpy(), xyz.cpu().numpy(), cnt.cpu().numpy()))
        assert torch.equal(voxel_down_sample(P64, voxel, device=dev), xyz[torch.argsort(keys)])
    report("float64 input", acc)


# ------------------------------------------------------------------------------------------------ a17 / a18 against the C++
@pytest.mark.parametrize("name", list(B.neighbor_cases()))
def test_radius_neighbors_vs_reference_edges(dev, oracle, name):
    from bufferx_b200 import ops
    q, s, qb, sb = (EDGES[f"nb_{name}_q"], EDGES[f"nb_{name}_s"]) + B.neighbor_cases()[name][2:4]
    r = B.neighbor_cases()[name][4]
    got = ops.radius_neighbors(cu(q, dev), cu(s, dev), qb, sb, r).cpu().numpy()
    out = B.check_neighbors(q, s, qb, sb, r, got, ref=EDGES[f"nb_{name}_ref"], oracle_rows=oracle.radius_neighbors(q, s, qb, sb, r))
    if name == "empty":
        assert got.shape == (len(q), 0)
    report(f"radius_neighbors {name}", out)


@pytest.mark.parametrize("name", list(B.subsample_cases()))
def test_grid_subsample_vs_reference_edges(dev, oracle, name):
    from bufferx_b200 import ops
    p, dl = EDGES[f"gs_{name}_p"], B.subsample_cases()[name][1]
    keys, xyz, cnt = ops.grid_subsample(cu(p, dev), dl)
    out = B.check_subsample(p, dl, keys.cpu().numpy(), xyz.cpu().numpy(), cnt.cpu().numpy(), EDGES[f"gs_{name}_ref"],
                            oracle.grid_subsample(p, dl))
    report(f"grid_subsample {name}", out)
