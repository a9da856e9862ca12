"""The checks of oracle/dropin_cases.py without a GPU: they accept correct answers (the literal fp32 kNN restatement,
numpy's float64 SVD rounded to fp32, a float64 port of bx_svd3's one-sided Jacobi rounded to fp32, the C oracle's ball
query, an exact gather) and reject subtly wrong ones: an fp32 Jacobi, a kNN that sums only the first 32 features or
returns a later duplicate, a ball query that tests <= or pads with the last hit, a gather that returns 0 out of range.
A check that accepts these mutants would let the same mistake in a kernel through tests/test_dropin_fp64_gpu.py.
The bounds are derived in the docstring of oracle/dropin_cases.py."""
import numpy as np
import pytest
import torch

from oracle import dropin_cases as D
from oracle import frontend_cases as F
from oracle.dropin_cases import merge, report


# ------------------------------------------------------------------------------------------------ SVD
def jacobi_svd3(A, dt):
    """bx_svd3.cuh's one-sided Jacobi restated in NumPy in the precision ``dt``, vectorised over the matrices (every
    operation rounds once in ``dt``: numpy has no FMA)."""
    A = np.asarray(A).astype(dt)
    n = len(A)
    w = A.transpose(0, 2, 1).copy()                           # w[:, j] = column j
    v = np.broadcast_to(np.eye(3, dtype=dt), (n, 3, 3)).copy()
    dot = lambda a, b: (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]
    done = np.zeros(n, bool)
    with np.errstate(all="ignore"):
        for _ in range(12):
            rotated = np.zeros(n, bool)
            for p, q in ((0, 1), (0, 2), (1, 2)):
                al, be, ga = dot(w[:, p], w[:, p]), dot(w[:, q], w[:, q]), dot(w[:, p], w[:, q])
                act = ~done & ~((ga == 0) | (np.abs(ga) <= dt(1e-15) * np.sqrt(al * be)))
                rotated |= act
                zeta = (be - al) / (dt(2) * np.where(act, ga, dt(1)))
                t = np.where(zeta >= 0, dt(1), dt(-1)) / (np.abs(zeta) + np.sqrt(dt(1) + zeta * zeta))
                c = dt(1) / np.sqrt(dt(1) + t * t)
                s = c * t
                c, s = np.where(act, c, dt(1))[:, None], np.where(act, s, dt(0))[:, None]
                for m in (w, v):
                    mp, mq = m[:, p].copy(), m[:, q].copy()
                    m[:, p], m[:, q] = c * mp - s * mq, s * mp + c * mq
            done |= ~rotated
    sv = np.sqrt(np.stack([dot(w[:, j], w[:, j]) for j in range(3)], 1))
    for a, b in ((0, 1), (1, 2), (0, 1)):
        sw = sv[:, a] < sv[:, b]
        sv[sw, a], sv[sw, b] = sv[sw, b], sv[sw, a].copy()
        for m in (w, v):
            m[sw, a], m[sw, b] = m[sw, b], m[sw, a].copy()
    with np.errstate(all="ignore"):
        u0 = np.where((sv[:, :1] > 0), w[:, 0] / np.where(sv[:, :1] > 0, sv[:, :1], 1), np.eye(3, dtype=dt)[0])
        u1 = w[:, 1].copy()
        for _ in range(2):
            u1 = u1 - dot(u0, u1)[:, None] * u0
        n1 = np.sqrt(dot(u1, u1))
        k = np.argmin(np.abs(u0), 1)                          # orth_complement: the least aligned axis, projected twice
        oc = np.eye(3, dtype=dt)[k]
        for _ in range(2):
            oc = oc - dot(u0, oc)[:, None] * u0
        oc = oc / np.sqrt(dot(oc, oc))[:, None]
        u1 = np.where((n1 > dt(1e-300))[:, None], u1 / np.where(n1 > 0, n1, 1)[:, None], oc)
    u2 = np.cross(u0, u1).astype(dt)
    u2 = np.where((dot(u2, w[:, 2]) < 0)[:, None], -u2, u2)
    Um = np.stack([u0, u1, u2], 2)
    return Um.astype(np.float32), sv.astype(np.float32), v.transpose(0, 2, 1).astype(np.float32)


@pytest.mark.parametrize("kind", D.SVD_KINDS)
def test_svd_checker_accepts_fp64(kind):
    """numpy's float64 SVD rounded to fp32, and the kernel's Jacobi run in float64 and rounded to fp32, both pass."""
    A = D.svd_case(kind, n=120, seed=3)
    u, s, vt = np.linalg.svd(A.astype(np.float64))
    acc = D.check_svd(A, u.astype(np.float32), s.astype(np.float32), vt.transpose(0, 2, 1).astype(np.float32))
    merge(acc, D.check_svd(A, *jacobi_svd3(A, np.float64)))
    report(f"svd checker accepts fp64, {kind}", acc)


@pytest.mark.parametrize("kind", ["random", "graded_cols", "graded_rows"])
def test_svd_checker_rejects_fp32_jacobi(kind):
    A = D.svd_case(kind, n=300, seed=4)
    with pytest.raises(AssertionError, match="S outside"):
        D.check_svd(A, *jacobi_svd3(A, np.float32))


def test_svd_checker_rejects_sign_inconsistent_pair():
    A = D.svd_case("random", n=50, seed=5)
    U, S, V = jacobi_svd3(A, np.float64)
    U[7, :, 1] *= -1                                            # still orthonormal and S unchanged
    with pytest.raises(AssertionError, match="reconstruction"):
        D.check_svd(A, U, S, V)


# ------------------------------------------------------------------------------------------------ kNN
def knn_mutant(ref, qry, first32=False, last_tie=False):
    """A kNN that sums only the first 32 features, or that keeps the last of equal minima."""
    r, q = torch.from_numpy(ref), torch.from_numpy(qry)
    if first32:
        r, q = r[..., :32].contiguous(), q[..., :32].contiguous()
    if not last_tie:
        return D.knn_fp32(r, q)
    d2 = torch.zeros(q.shape[:2] + r.shape[1:2])
    for c in range(q.shape[2]):
        t = q[:, :, None, c] - r[:, None, :, c]
        d2 = d2 + t * t
    Nr = r.shape[1]
    idx = Nr - 1 - torch.argmin(d2.flip(-1), -1)
    return torch.sqrt(d2.gather(-1, idx[..., None])[..., 0]), idx


@pytest.mark.parametrize("kind", D.KNN_KINDS)
@pytest.mark.parametrize("Dim", [1, 3, 31, 33, 65])
def test_knn_checker_accepts_literal(kind, Dim):
    acc = {}
    for B, Nr, Nq in ((1, 1, 5), (3, 65, 63), (2, 130, 20)):
        ref, qry = D.knn_case(kind, B, Nr, Nq, Dim, seed=Dim + Nr)
        dist, idx = D.knn_fp32(ref, qry)
        merge(acc, D.check_knn(ref, qry, dist, idx))
    if kind == "overflow":
        assert acc["knn_all_inf"] > 0
    report(f"knn checker accepts the literal arithmetic, {kind}, D={Dim}", acc)


def test_knn_fp32_equals_numpy_restatement():
    """knn_fp32 (torch, chunked) equals the same arithmetic in NumPy, whose sqrt is correctly rounded as sqrtf is on the
    GPU: torch's CPU fp32 sqrt is an ulp off on some of these distances, so knn_fp32 takes it through float64."""
    rng = np.random.default_rng(303)
    for Dim, Nr, Nq in ((3, 5000, 2000), (70, 300, 200)):
        ref = rng.standard_normal((2, Nr, Dim)).astype(np.float32)
        qry = rng.standard_normal((2, Nq, Dim)).astype(np.float32)
        dist, idx = D.knn_fp32(ref, qry)
        for b in range(2):
            d2 = np.zeros((Nq, Nr), np.float32)
            for c in range(Dim):
                t = qry[b][:, None, c] - ref[b][None, :, c]
                d2 = d2 + t * t
            i = np.argmin(d2, 1)
            assert np.array_equal(idx[b].numpy(), i)
            assert np.array_equal(dist[b].numpy().view(np.int32), np.sqrt(d2[np.arange(Nq), i]).view(np.int32))


@pytest.mark.parametrize("kind", ["mixed", "offset"])
def test_knn_checker_rejects_first32_and_last_duplicate(kind):
    ref, qry = D.knn_case(kind, 2, 130, 20, 40, seed=1)
    dist, idx = knn_mutant(ref, qry, first32=True)
    with pytest.raises(AssertionError):
        D.check_knn(ref, qry, dist, idx)
    with pytest.raises(AssertionError, match="decided arg-min"):         # float64 alone catches it as well
        D.check_knn(ref, qry, dist, idx, literal=False)
    dist, idx = knn_mutant(ref, qry, last_tie=True)
    with pytest.raises(AssertionError):
        D.check_knn(ref, qry, dist, idx)
    with pytest.raises(AssertionError, match="later copy"):
        D.check_knn(ref, qry, dist, idx, literal=False)


def test_knn_lattice_has_float64_ties():
    ref, qry = D.knn_case("lattice", 2, 200, 100, 4, seed=2)
    r, q = ref.astype(np.float64), qry.astype(np.float64)
    d = ((q[:, :, None] - r[:, None]) ** 2).sum(-1)
    s = np.sort(d, -1)
    assert (s[..., 0] == s[..., 1]).mean() > 0.3


def test_radius_decision_checker():
    rng = np.random.default_rng(0)
    tgt = rng.uniform(-1, 1, (400, 3)).astype(np.float32)
    src = (tgt[:300] + rng.normal(scale=0.03, size=(300, 3))).astype(np.float32)
    dist, _ = D.knn_fp32(tgt[None], src[None])
    out = D.check_radius_decision(dist, src, tgt, 0.04)
    assert 0 < out["vs_matches"] < 300
    with pytest.raises(AssertionError):
        D.check_radius_decision(dist * 1.05, src, tgt, 0.04)


# ------------------------------------------------------------------------------------------------ ball query
def ball_query_np(xyz, qry, radius, nsample, le=False, pad_last=False):
    """pointnet2 ball_query restated in fp32 NumPy (d2 = ((dx dx) + (dy dy)) + dz dz, hit d2 < r^2); the mutants test
    <= or pad with the last hit."""
    r2 = np.float32(np.float32(radius) * np.float32(radius))
    idx = np.zeros((len(qry), nsample), np.int32)
    for j, q in enumerate(qry):
        d = (q[None] - xyz).astype(np.float32)
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        hits = np.flatnonzero(d2 <= r2 if le else d2 < r2)[:nsample]
        if len(hits):
            idx[j, :len(hits)] = hits
            idx[j, len(hits):] = hits[-1] if pad_last else hits[0]
    return idx


@pytest.mark.parametrize("nsample", [1, 31, 33])
def test_ball_query_checker(oracle, nsample):
    acc = {}
    for kind in ("exact", "counts"):
        pts, kp, r = F.patch_case(kind, n=600, k=24, P=nsample, seed=nsample)
        want, _ = oracle.ball_query(pts, kp, r, nsample)
        assert np.array_equal(ball_query_np(pts, kp, r, nsample), want)
        merge(acc, D.check_ball_query(pts, kp, r, want))
        merge(acc, D.check_ball_query(pts[None].repeat(2, 0), kp[None].repeat(2, 0), r, want[None].repeat(2, 0)))
        if kind == "exact":
            with pytest.raises(AssertionError, match="decided miss"):
                D.check_ball_query(pts, kp, r, ball_query_np(pts, kp, r, nsample, le=True))
        elif nsample > 1:
            with pytest.raises(AssertionError, match="padding"):
                D.check_ball_query(pts, kp, r, ball_query_np(pts, kp, r, nsample, pad_last=True))
    report(f"ball query checker, nsample {nsample}", acc)


def test_batched_ball_query_checker_keeps_clouds_apart(oracle):
    """A row of cloud 1 answered with cloud 0's points fails."""
    pts, kp, r = F.patch_case("counts", n=600, k=24, P=16, seed=3)
    other = pts[np.random.default_rng(0).permutation(len(pts))]
    xyz, q = np.stack([pts, other]), np.stack([kp, kp])
    idx = np.stack([oracle.ball_query(pts, kp, r, 16)[0]] * 2)
    with pytest.raises(AssertionError):
        D.check_ball_query(xyz, q, r, idx)


# ------------------------------------------------------------------------------------------------ gather
def test_gather_checker():
    rng = np.random.default_rng(1)
    f = rng.standard_normal((2, 3, 50)).astype(np.float32)
    f.view(np.int32)[0, 0, :4] = [0x7FC12345, np.int32(-2147483648), 1, 0x7F800000]   # NaN payload, -0.0, subnormal, inf
    idx = rng.integers(0, 50, (2, 40)).astype(np.int32)
    idx[:, :4] = [0, 1, 2, 3]
    idx[1, 10:14] = [-1, 50, 2147483647, -2147483648]
    good = D.gather_want(f, idx).view(np.float32)
    out = D.check_gather(f, idx, good)
    assert out["gather_out_of_range"] == 4
    zero = good.copy()
    zero[1, :, 10:14] = 0.0
    with pytest.raises(AssertionError):
        D.check_gather(f, idx, zero)
    quiet = good.copy()
    quiet.view(np.int32)[0, 0, 0] = 0x7FC00000                  # a NaN, but not the copied payload
    with pytest.raises(AssertionError):
        D.check_gather(f, idx, quiet)
