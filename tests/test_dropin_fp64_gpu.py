"""The drop-in modules under dropin/ on the GPU against float64, on edge inputs, through the modules exactly as the
reference imports them (knn_cuda, torch_batch_svd, pointnet2_ops.pointnet2_utils).

kNN at feature lengths across the kernel's 32-column stages and row counts across its 64-row tiles, bit for bit against
the literal fp32 arithmetic and held to float64 (decided arg-mins, margins, first of equal rows, distance bound); the
reference's get_matching_indices and mutual_matching call shapes.  The 3x3 SVD on the case catalogue and batch sizes
around its 128-thread blocks.  Gathers as bit copies with out-of-range indices.  The ball query on both routes, at
nsample around the 32-lane batches, r = 0 and the launch splits of the shared-memory route.  The checks and their
derived bounds are in oracle/dropin_cases.py (pinned without a GPU by tests/test_dropin_fp64_cpu.py); the largest
ratios are printed with -s and recorded in DESIGN.md section 7."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import dropin_cases as D
from oracle import frontend_cases as F
from oracle.dropin_cases import merge, report
from oracle.pose_cases import desc_set

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


def cu(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


# ------------------------------------------------------------------------------------------------ kNN
def _knn(mods, ref, qry):
    dist, idx = mods[1].KNN(k=1, transpose_mode=True)(ref, qry)
    assert dist.dtype == torch.float32 and idx.dtype == torch.int64
    assert tuple(dist.shape) == (qry.shape[0], qry.shape[1], 1) and tuple(idx.shape) == dist.shape
    return dist[..., 0], idx[..., 0]


KNN_D = [1, 3, 31, 32, 33, 63, 64, 65, 100, 128]


@pytest.mark.parametrize("Dim", KNN_D)
def test_knn_feature_stages(dev, mods, Dim):
    """Every case kind at Nr, Nq across the 64-row tiles, B = 1 and 3."""
    acc = {}
    sizes = [(1, 1, 1), (3, 63, 64), (1, 64, 65), (3, 65, 63), (1, 4097, 65), (3, 65, 4097)]
    for kind in D.KNN_KINDS:
        for B, Nr, Nq in sizes:
            ref, qry = D.knn_case(kind, B, Nr, Nq, Dim, seed=Dim * 7 + Nr + Nq)
            r, q = cu(ref, dev), cu(qry, dev)
            dist, idx = _knn(mods, r, q)
            merge(acc, D.check_knn(r, q, dist, idx))
    assert acc["knn_all_inf"] > 0
    report(f"knn D={Dim}", acc)


@pytest.mark.parametrize("Dim", [33, 100])
def test_knn_large_tiles(dev, mods, Dim):
    """Nr = Nq = 4097 (65 x 65 tiles) with the mixed edge rows."""
    ref, qry = D.knn_case("mixed", 1, 4097, 4097, Dim, seed=Dim)
    r, q = cu(ref, dev), cu(qry, dev)
    dist, idx = _knn(mods, r, q)
    report(f"knn 4097 x 4097, D={Dim}", D.check_knn(r, q, dist, idx))


def test_knn_many_tiny_problems(dev, mods):
    """B in the thousands (grid.z) on tiny problems, every kind."""
    acc = {}
    for kind, (B, Nr, Nq, Dim) in zip(D.KNN_KINDS, [(4000, 13, 5, 33), (3000, 7, 9, 3), (5000, 12, 3, 3), (2000, 5, 6, 40)]):
        ref, qry = D.knn_case(kind, B, Nr, Nq, Dim, seed=B)
        r, q = cu(ref, dev), cu(qry, dev)
        dist, idx = _knn(mods, r, q)
        merge(acc, D.check_knn(r, q, dist, idx))
    report("knn B in the thousands", acc)


def test_knn_get_matching_indices_shape(dev, mods):
    """BUFFERX.get_matching_indices: the C2 source moved by its ground-truth pose ([1, N, 3] on the device, as the
    reference's transform), kNN into the target, and the decision dist < search_voxel_size (0.0375, 0.075) held to
    float64 outside its margin."""
    from bufferx_b200.synth import make_pair
    data = make_pair("C2", 0)
    src = torch.from_numpy(data["src_fds_pcd"].astype(np.float32)).to(dev)
    tgt = torch.from_numpy(data["tgt_fds_pcd"].astype(np.float32)).to(dev)
    T = torch.from_numpy(np.asarray(data["relt_pose"], np.float32)).to(dev)
    src = (src @ T[:3, :3].T + T[:3, 3]).contiguous()
    dist, idx = _knn(mods, tgt[None], src[None])
    acc = D.check_knn(tgt[None], src[None], dist, idx)
    for vs in (0.0375, 0.075):
        merge(acc, D.check_radius_decision(dist, src, tgt, vs))
    assert acc["vs_matches"] > 0
    report("knn get_matching_indices (C2 seed 0)", acc)


@pytest.mark.parametrize("K", [1500, 3000])
def test_knn_mutual_matching_shape(dev, mods, K):
    """BUFFERX.mutual_matching: [1, K, 32] both ways, indices equal to the production ops.mutual_nn (snn, tnn) bit for
    bit, and each side held to float64."""
    from bufferx_b200 import ops
    a, b = desc_set(K, K - 7, seed=K)
    ta, tb = cu(a, dev), cu(b, dev)
    ds, s_idx = _knn(mods, tb[None], ta[None])
    dt, t_idx = _knn(mods, ta[None], tb[None])
    _, _, _, snn, tnn = ops.mutual_nn(ta, tb, want_nn=True)
    assert torch.equal(s_idx[0], snn[:K].long()) and torch.equal(t_idx[0], tnn[:K - 7].long())
    acc = D.check_knn(tb[None], ta[None], ds, s_idx)
    merge(acc, D.check_knn(ta[None], tb[None], dt, t_idx))
    report(f"knn mutual_matching K={K}", acc)


def test_knn_refusals(dev, mods):
    """B = 65536 and Nr = 65535 * 64 + 1 raise BufferXError (not a launch failure); the next call still works."""
    from bufferx_b200.ops import BufferXError
    x = torch.rand((65536, 1, 1), device=dev)
    with pytest.raises(BufferXError, match="B=65536"):
        _knn(mods, x, x)
    r = torch.rand((1, 65535 * 64 + 1, 1), device=dev)
    with pytest.raises(BufferXError, match="ref rows"):
        _knn(mods, r, r[:, :5])
    dist, idx = _knn(mods, r[:, :65535 * 64], r[:, :5])
    assert torch.equal(idx[0], torch.arange(5, device=dev)) and bool((dist == 0).all())
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ SVD
def _svd(mods, A):
    U, S, V = mods[2].svd(A)
    assert U.dtype == S.dtype == V.dtype == torch.float32
    assert tuple(U.shape) == tuple(V.shape) == (A.shape[0], 3, 3) and tuple(S.shape) == (A.shape[0], 3)
    return U, S, V


@pytest.mark.parametrize("B", [0, 1, 127, 128, 129, 100000])
def test_svd_batch_sizes(dev, mods, B):
    """Batch sizes around the 128-thread blocks, the catalogue cycled; two runs bit-identical."""
    A = np.concatenate([D.svd_case(k, n=max(1, B // len(D.SVD_KINDS) + 1), seed=B) for k in D.SVD_KINDS])
    A = A[np.random.default_rng(B).permutation(len(A))[:B]]
    At = cu(A, dev)
    U, S, V = _svd(mods, At)
    acc = D.check_svd(A, U, S, V)
    U2, S2, V2 = _svd(mods, At)
    assert all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in ((U, U2), (S, S2), (V, V2)))
    report(f"svd B={B}", acc)


def test_svd_non_contiguous(dev, mods):
    A = cu(np.concatenate([D.svd_case(k, n=40, seed=9) for k in D.SVD_KINDS]), dev)
    At = A.transpose(1, 2)
    assert not At.is_contiguous()
    got = _svd(mods, At)
    want = _svd(mods, At.contiguous())
    assert all(torch.equal(x, y) for x, y in zip(got, want))
    report("svd non-contiguous", D.check_svd(At.contiguous().cpu().numpy(), *got))


# ------------------------------------------------------------------------------------------------ gather / group
def test_gather_and_group_bit_copies(dev, mods):
    """C = 1 and N = 1, K not a multiple of 256, [B,M,S] with S = 1 and large M*S, non-contiguous features, NaN payloads,
    -0.0 and subnormals in the features, and indices -1, N, INT32_MAX, INT32_MIN (NaN 0x7fc00000, neighbours intact)."""
    p2 = mods[0]
    rng = np.random.default_rng(0)
    acc = {}

    def feats(B, C, N):
        f = rng.standard_normal((B, C, N)).astype(np.float32)
        bits = f.reshape(-1).view(np.int32)
        sel = rng.choice(bits.size, min(bits.size, 64), replace=False)
        bits[sel] = rng.choice([0x7FC12345, 0x7F800001, -2147483648, 1, 0x007FFFFF, -8388608], len(sel)).astype(np.int32)
        return f

    def idx_of(shape, N, bad=True):
        i = rng.integers(0, N, shape).astype(np.int64)
        if bad:
            flat = i.reshape(i.shape[0], -1)
            for j, v in enumerate((-1, N, 2 ** 31 - 1, -2 ** 31)):
                if flat.shape[1] > 2 * j + 1:
                    flat[:, 2 * j + 1] = v
        return i.astype(np.int32)

    for B, C, N, M in ((1, 1, 1, 1), (2, 1, 1, 7), (3, 5, 1000, 255), (2, 3, 700, 257), (1, 7, 4000, 1000), (4, 2, 50, 513)):
        f, i = feats(B, C, N), idx_of((B, M), N)
        out = p2.gather_operation(cu(f, dev), cu(i, dev))
        assert tuple(out.shape) == (B, C, M)
        merge(acc, D.check_gather(f, i, out))
    for B, C, N, M, S in ((2, 3, 500, 40, 1), (1, 4, 20000, 1500, 512), (3, 1, 1, 5, 3), (2, 6, 900, 33, 17)):
        f, i = feats(B, C, N), idx_of((B, M, S), N)
        out = p2.grouping_operation(cu(f, dev), cu(i, dev))
        assert tuple(out.shape) == (B, C, M, S)
        merge(acc, D.check_gather(f, i, out))
    f = feats(3, 400, 6)                                       # non-contiguous: [B, N, C] transposed to [B, C, N]
    ft = cu(f, dev).transpose(1, 2)
    assert not ft.is_contiguous()
    i = idx_of((3, 300), 400)
    merge(acc, D.check_gather(ft.cpu(), i, p2.gather_operation(ft, cu(i, dev))))
    gi = idx_of((3, 20, 9), 400)
    merge(acc, D.check_gather(ft.cpu(), gi, p2.grouping_operation(ft, cu(gi, dev))))
    assert acc["gather_out_of_range"] > 0
    report("gather / group", acc)


# ------------------------------------------------------------------------------------------------ ball query
def _far(pts, n_total):
    """pts with points appended 1e4 m away (never hit) up to n_total points."""
    extra = np.random.default_rng(n_total).uniform(-1, 1, (n_total - len(pts), 3)) + 1e4
    return np.concatenate([pts, extra]).astype(np.float32)


@pytest.mark.parametrize("nsample", [1, 31, 32, 33, 100, 512])
def test_ball_query_nsample_both_routes(dev, mods, nsample):
    """Balls with nsample - 1, nsample and nsample + 1 hits; N <= 4096 (shared memory) and the same cloud grown past
    4096 by far points (global) give equal rows, each held to float64; r = 0 gives all-zero rows, on points too."""
    p2 = mods[0]
    acc = {}
    k = 3 * max(1, min(16, 3900 // (3 * (nsample + 1))))
    pts, kp, r = F.patch_case("counts", n=3900, k=k, P=nsample, seed=nsample)
    pts = pts[:4000]
    assert len(pts) <= 4096
    kp = np.concatenate([kp, pts[:5]]).astype(np.float32)      # queries on cloud points
    x, q = cu(pts, dev), cu(kp, dev)
    small = p2.ball_query(r, nsample, x[None], q[None])
    big = p2.ball_query(r, nsample, cu(_far(pts, 5000), dev)[None], q[None])
    assert torch.equal(small, big), "shared-memory and global routes differ"
    merge(acc, D.check_ball_query(x, q, r, small[0]))
    counts = (small[0, :, 1:] > small[0, :, :-1]).long().cumprod(1).sum(1) + 1
    assert bool((counts[:k] == nsample).any()) and (nsample == 1 or bool((counts[:k] == nsample - 1).any()))
    for xx in (x, cu(_far(pts, 5000), dev)):
        z = p2.ball_query(0.0, nsample, xx[None], q[None])
        assert bool((z == 0).all()), "r = 0 must give all-zero rows"
    report(f"ball query nsample {nsample}", acc)


@pytest.mark.parametrize("B,N,M", [(1, 4096, 20000), (1, 4097, 20000), (7, 300, 1600), (1056, 60, 40), (1057, 60, 40),
                                   (65535, 4, 2), (300, 4097, 5)])
def test_ball_query_launch_splits(dev, mods, B, N, M):
    """The shared-memory route's CTA striding (B = 1, M = 20000; B = 7 where ceil(1056 / B) = 151 does not divide the
    200 per-cloud CTAs), one CTA per cloud (B = 1056, 1057), B = 65535 and the global route with many clouds; every row
    to float64."""
    p2 = mods[0]
    rng = np.random.default_rng(B + N + M)
    xyz = rng.uniform(-1, 1, (B, N, 3)).astype(np.float32)
    qry = np.concatenate([xyz[:, :1], rng.uniform(-1, 1, (B, max(0, M - 1), 3))], 1)[:, :M].astype(np.float32)
    x, q = cu(xyz, dev), cu(qry, dev)
    r = 0.9 if N <= 8 else 0.25
    got = p2.ball_query(r, 16, x, q)
    assert tuple(got.shape) == (B, M, 16)
    acc = D.check_ball_query(x, q, r, got)
    assert acc["bq_rows"] == B * M
    report(f"ball query B={B} N={N} M={M}", acc)


def test_ball_query_refusal(dev, mods):
    from bufferx_b200.ops import BufferXError
    x = torch.rand((65536, 3, 3), device=dev)
    with pytest.raises(BufferXError, match="B=65536"):
        mods[0].ball_query(0.5, 4, x, x)
    torch.cuda.synchronize()
