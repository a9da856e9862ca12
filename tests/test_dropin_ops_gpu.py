"""The drop-in modules under dropin/ (pointnet2_ops.pointnet2_utils, knn_cuda, torch_batch_svd) on the GPU, at the
reference's call shapes, against the oracle: FPS and ball query bit for bit, gather / group as exact copies, k = 1
nearest neighbour index and distance bits, and the 3x3 SVD against numpy's float64 SVD and against the LRF's z axis."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import dropin_cases as DC

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DROPIN = os.path.join(ROOT, "dropin")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    if DROPIN not in sys.path:
        sys.path.insert(0, DROPIN)
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def mods(dev):
    import knn_cuda
    import torch_batch_svd
    from pointnet2_ops import pointnet2_utils
    for m in (knn_cuda, torch_batch_svd, pointnet2_utils):
        assert os.path.realpath(m.__file__).startswith(os.path.realpath(DROPIN)), m.__file__
    return pointnet2_utils, knn_cuda, torch_batch_svd


@pytest.fixture(scope="module")
def c2(oracle):
    """The C2 seed-0 source cloud (20000 points), its 1500 golden FPS key-points and the golden scale-0 radius."""
    from bufferx_b200.synth import make_pair
    g = np.load(os.path.join(ROOT, "tests", "golden", "c2_seed0.npz"))
    pts = make_pair("C2", 0)["src_fds_pcd"].astype(np.float32)
    kpts = np.ascontiguousarray(pts[g["s_fps"][:1500]])
    return pts, kpts, float(np.float32(g["des_r"][0]))


def cu(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


# ------------------------------------------------------------------------------------------------ FPS, gather
@pytest.mark.parametrize("B", [1, 3, 20])
def test_furthest_point_sample_equals_oracle(dev, mods, oracle, B):
    p2 = mods[0]
    rng = np.random.default_rng(B)
    xyz = (rng.standard_normal((B, 3000, 3)) * [2.0, 1.0, 0.5]).astype(np.float32)
    got = p2.furthest_point_sample(cu(xyz, dev), 256)
    assert got.dtype == torch.int32 and tuple(got.shape) == (B, 256)
    want = np.stack([oracle.fps(x, 256) for x in xyz])
    assert np.array_equal(got.cpu().numpy(), want)


def test_gather_and_group_equal_torch_gather(dev, mods):
    p2 = mods[0]
    rng = np.random.default_rng(5)
    feat = cu(rng.standard_normal((3, 7, 1000)).astype(np.float32), dev)
    idx = cu(rng.integers(0, 1000, (3, 150), dtype=np.int32), dev)
    got = p2.gather_operation(feat, idx)
    assert torch.equal(got, torch.gather(feat, 2, idx.long()[:, None, :].expand(-1, 7, -1)))
    gidx = cu(rng.integers(0, 1000, (3, 40, 17), dtype=np.int32), dev)
    got = p2.grouping_operation(feat, gidx)
    want = torch.gather(feat, 2, gidx.long().reshape(3, 1, -1).expand(-1, 7, -1)).reshape(3, 7, 40, 17)
    assert tuple(got.shape) == (3, 7, 40, 17) and torch.equal(got, want)


# ------------------------------------------------------------------------------------------------ ball query
def _ball_query_vs_oracle(p2, oracle, dev, xyz, qry, radius, nsample):
    got = p2.ball_query(radius, nsample, cu(xyz, dev), cu(qry, dev))
    assert got.dtype == torch.int32 and tuple(got.shape) == (xyz.shape[0], qry.shape[1], nsample)
    got = got.cpu().numpy()
    for b in range(xyz.shape[0]):
        want, _ = oracle.ball_query(xyz[b], qry[b], radius, nsample)
        assert np.array_equal(got[b], want), f"cloud {b}: {int((got[b] != want).any(1).sum())} rows differ"
    return got


def test_ball_query_one_large_cloud(dev, mods, oracle, c2):
    """select_patches (patch_embedder.py:99): B = 1, the C2 cloud, 1500 FPS key-points, the golden radius, 512 samples."""
    pts, kpts, r = c2
    got = _ball_query_vs_oracle(mods[0], oracle, dev, pts[None], kpts[None], r, 512)
    assert (got[0, :, 1] != got[0, :, 0]).mean() > 0.5           # most balls hold more than one point


def test_ball_query_many_small_clouds(dev, mods, oracle, c2):
    """sphere_query (common.py:442): 1500 LRF-normalised patches of 512 points against the 420 voxel centres, 10 samples."""
    pts, kpts, r = c2
    _, patches = oracle.select_patches(pts, None, kpts, r, 512)
    delta, _, _ = oracle.lrf(patches, r, False)
    vox = np.broadcast_to(oracle.voxel_table(), (len(delta), 420, 3))
    _ball_query_vs_oracle(mods[0], oracle, dev, delta, vox, np.float32(0.8 / 3), 10)


@pytest.mark.parametrize("N", [1, 31, 33, 100, 4097])
@pytest.mark.parametrize("B", [1, 5])
def test_ball_query_edge_cases(dev, mods, oracle, N, B):
    """Empty balls (all-zero rows), fewer hits than nsample (padding with the first hit), the first hit at index 0, and
    N not a multiple of 32, on both sides of the shared-memory cloud limit (4096 points)."""
    rng = np.random.default_rng(N * 10 + B)
    xyz = rng.uniform(-1, 1, (B, N, 3)).astype(np.float32)
    qry = np.concatenate([xyz[:, :1], rng.uniform(-1, 1, (B, 30, 3)), np.full((B, 3, 3), 50.0)], axis=1).astype(np.float32)
    got = _ball_query_vs_oracle(mods[0], oracle, dev, xyz, qry, 0.3, 16)
    assert (got[:, 0, 0] == 0).all() and (got[:, -3:] == 0).all()


# ------------------------------------------------------------------------------------------------ kNN
@pytest.mark.parametrize("D,B,Nr,Nq", [(3, 3, 5000, 2000), (32, 2, 1500, 1500), (32, 1, 100, 1), (5, 2, 65, 70)])
def test_knn_equals_oracle_arithmetic(dev, mods, oracle, D, B, Nr, Nq):
    KNN = mods[1].KNN
    rng = np.random.default_rng(D * 100 + B)
    ref = rng.standard_normal((B, Nr, D)).astype(np.float32)
    ref[:, Nr // 2:Nr // 2 + 3] = ref[:, 1:4]                      # exact duplicate rows: the first one must win
    qry = rng.standard_normal((B, Nq, D)).astype(np.float32)
    qry[:, :min(3, Nq)] = ref[:, Nr // 2:Nr // 2 + min(3, Nq)]
    dist, idx = KNN(k=1, transpose_mode=True)(cu(ref, dev), cu(qry, dev))
    assert dist.dtype == torch.float32 and idx.dtype == torch.int64
    assert tuple(dist.shape) == (B, Nq, 1) and tuple(idx.shape) == (B, Nq, 1)
    dist, idx = dist[..., 0].cpu().numpy(), idx[..., 0].cpu().numpy()
    for b in range(B):
        _, _, snn, _ = oracle.mutual_nn(qry[b], ref[b])
        assert np.array_equal(idx[b], snn)
    want_d, want_i = DC.knn_fp32(ref, qry)
    assert np.array_equal(idx, want_i.numpy()) and np.array_equal(dist.view(np.int32), want_d.numpy().view(np.int32))
    assert (idx[:, :min(3, Nq)] == np.arange(1, 1 + min(3, Nq))).all()


# ------------------------------------------------------------------------------------------------ SVD
def test_svd_against_numpy_float64(dev, mods):
    """The whole case catalogue of oracle/dropin_cases.py held to numpy's float64 SVD by check_svd: S within
    u s + 64 u53 s_max, orthonormality within 3u, reconstruction, U/V pairing, vectors and cluster projectors (bounds
    derived there; an fp32 Jacobi fails them)."""
    A = np.concatenate([DC.svd_case(k, n=200, seed=11) for k in DC.SVD_KINDS])
    U, S, V = mods[2].svd(cu(A, dev))
    out = DC.check_svd(A, U, S, V)
    assert out["svd_vectors"] > 2000 and out["svd_projectors"] > 500
    DC.report("svd catalogue", out)


def test_cal_z_axis_from_dropin_svd_matches_lrf(dev, mods, oracle, c2):
    """cal_Z_axis (common.py:709-726) built with the drop-in svd on oracle patches: z = u[:,:,-1], flipped when
    -z . centre < 0, normalised -- the oracle LRF's z axis where the eigen-gap and the sign margin are clear."""
    pts, kpts, r = c2
    _, patches = oracle.select_patches(pts, None, kpts, r, 512)
    _, _, _, z_or = oracle.lrf(patches, r, False, want_z=True)
    f = oracle.lrf_fp64(patches, r, False)
    p = cu(patches, dev)
    center = p[:, -1, :]
    local = p - center[:, None, :]
    u, _, _ = mods[2].svd(torch.matmul(local.transpose(-1, -2), local))
    z = u[:, :, -1]
    mask = (torch.sum(-z * center, dim=1) < 0).float().unsqueeze(1)
    z = z * (1 - mask) - z * mask
    z = (z / torch.norm(z, dim=1, keepdim=True)).cpu().numpy()
    clear = (f["gap"] > 1e-2 * f["lam"][:, 2]) & (f["margin"] > 1e-3 * np.linalg.norm(patches[:, -1], axis=1))
    assert clear.mean() > 0.5
    assert np.abs(z - z_or)[clear].max() <= 1e-4


# ------------------------------------------------------------------------------------------------ refusals
def test_unsupported_inputs_raise(dev, mods):
    from bufferx_b200.ops import BufferXError
    p2, knn, tbs = mods
    x = torch.rand((1, 100, 3), device=dev)
    with pytest.raises(NotImplementedError):
        knn.KNN(k=2, transpose_mode=True)
    with pytest.raises(NotImplementedError):
        knn.KNN(k=1, transpose_mode=False)
    with pytest.raises(NotImplementedError):
        knn.KNN(k=1, transpose_mode=True)(x.clone().requires_grad_(True), x)
    with pytest.raises(NotImplementedError):
        p2.ball_query(0.1, 8, x.clone().requires_grad_(True), x)
    with pytest.raises(NotImplementedError):
        tbs.svd(torch.rand((4, 3, 3), device=dev, requires_grad=True))
    with pytest.raises(NotImplementedError):
        tbs.svd(torch.rand((4, 4, 4), device=dev))
    with pytest.raises(BufferXError):
        p2.furthest_point_sample(x.cpu(), 10)
    with pytest.raises(BufferXError):
        knn.KNN(k=1, transpose_mode=True)(x.cpu(), x.cpu())
    with pytest.raises(BufferXError):
        tbs.svd(torch.rand((4, 3, 3)))
    with pytest.raises(BufferXError, match="524288"):
        p2.furthest_point_sample(torch.rand((1, 524289, 3), device=dev), 4)
