"""Edge inputs of the drop-in modules under dropin/ (knn_cuda.KNN -> bx_knn1, torch_batch_svd.svd -> bx_svd3,
pointnet2_ops gather_operation / grouping_operation -> bx_gather_channels, ball_query -> bx_ball_query_batched) and the
float64 checks they are held to, shared by tests/test_dropin_fp64_cpu.py (which shows every check rejecting a subtly
wrong implementation) and tests/test_dropin_fp64_gpu.py (the kernels).  The ball query reuses
frontend_cases.check_ball_query and the kNN arg-min reuses the matching margin of pose_cases._nn_side.

Bounds (u = 2^-24, u53 = 2^-53, TINY = 2^-150 = half the fp32 subnormal spacing, the absolute rounding error of an fp32
result below the normal range):

* kNN.  The kernel sums fl(q_c - r_c)^2 over D features in order from +0 without FMA: ``knn_fp32`` restates that
  arithmetic literally and the kernel must equal it bit for bit (index: the first fp32 minimum; distance: sqrtf of it).
  In float64, the fp32 sum is within KN (D + 3) u d64 of d64 (non-negative terms: the error is relative to d itself;
  KN = 4 of slack), so a query's arg-min is decided when the float64 gap between the best and the second best exceeds
  both errors: decided arg-mins are float64's first minimum, the others lie within the margin (pose_cases._nn_side with
  C = D).  Bitwise-equal rows give bitwise-equal distances, so the first of them must win.  The kernel's fp32 minimum
  and float64's minimum d64 are both within the margin of d64, so dist = fl(sqrt(fl32 d)) is within
  (KN (D + 3) / 2 + 1) u sqrt(d64) + 1e-15 of sqrt(d64) (1e-15 = sqrt of the margin's absolute floor 1e-30, which
  covers underflow of the squares).  Squared differences beyond fp32's range: the contract is the literal fp32
  arithmetic -- such distances are +inf, and a query whose every distance is +inf takes the first ref row (index 0,
  dist +inf); those queries are outside the float64 checks.
* SVD, against numpy's float64 SVD of the fp32 input (s64, U64, V64).  The kernel's fp64 Jacobi and numpy are each
  backward stable (KS/2 u53 s_max, KS = 64 for both together); the fp32 rounding of the outputs adds u s (or TINY):
  |S - s64| <= u s64 + (1 + u) KS u53 s_max + TINY.  U and V are fp64-orthonormal columns rounded entrywise by u, so
  |U^T U - I| <= 2u + u^2 <= 3u (Cauchy-Schwarz over the rows).  Reconstruction ||U diag(S) V^T - A||_F (evaluated in
  float64) <= (3u + 4u^2 + 2 KS u53) ||A||_F + 2 TINY: one u ||A||_F per rounded factor, KS u53 for the factorisation
  and its float64 evaluation.  Pairing ||A v_i - s_i u_i|| <= u (s_max + 2 s_i + u s_i) + 2 KS u53 s_max + 2 TINY: a
  sign-inconsistent (u_i, v_i) leaves 2 s_i.  Vectors (Wedin): a singular value isolated by gap g has u_i, v_i within
  KS u53 s_max / g + 2u of float64's (up to sign, entrywise); values closer than 2^10 KS u53 s_max form a cluster, whose
  projector U_c U_c^T (and V_c V_c^T) is within KS u53 s_max / g_c + 3u of float64's, g_c the distance to the rest.
  An fp32 Jacobi misses the S bound by orders of magnitude (tests/test_dropin_fp64_cpu.py).
* Gather.  A copy: equal bits (NaN payloads, -0.0, subnormals); an index outside [0, N) gives the NaN 0x7fc00000.
* Ball query.  frontend_cases.check_ball_query on every row.

Each check returns a dict of ratios (floats, the largest is kept by ``merge``) and counts (ints, summed)."""
import numpy as np
import torch

from oracle import oracle as O
from oracle.frontend_cases import check_ball_query  # noqa: F401  (re-exported for the tests)
from oracle.pose_cases import KN, _nn_side, merge  # noqa: F401

F32 = np.float32
U = 2.0 ** -24
U53 = 2.0 ** -53
TINY = 2.0 ** -150
KS = 64.0
NAN_BITS = 0x7FC00000


def report(name, out):
    ratios = {k: v for k, v in out.items() if isinstance(v, float)}
    counts = {k: v for k, v in out.items() if isinstance(v, (int, np.integer))}
    print(f"\n[dropin-fp64] {name}: " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items())
          + (" | " + ", ".join(f"{k} {v}" for k, v in counts.items()) if counts else ""))


def _t(a, dev=None):
    t = a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))
    return t if dev is None else t.to(dev)


# ------------------------------------------------------------------------------------------------ kNN
KNN_KINDS = ("mixed", "lattice", "offset", "overflow")


def knn_case(kind, B, Nr, Nq, D, seed=0):
    """(ref [B,Nr,D], qry [B,Nq,D]) fp32.  'mixed': normal rows with exact duplicates in different 64-row tiles, pairs
    equal in the first 32 features and different after them, rows one ulp apart and zero rows, each with a query on it;
    'lattice': small integers, so every distance is exact and queries sit exactly between two refs (float64 ties);
    'offset': the mixed rows scaled to 1 m around a 1e4 m offset; 'overflow': rows near +-1e20 whose squared
    differences overflow fp32, with some queries beyond every ref (all distances +inf)."""
    rng = np.random.default_rng(seed)
    if kind == "lattice":
        ref = rng.integers(-2, 3, (B, Nr, D)).astype(np.float64)
        qry = rng.integers(-2, 3, (B, Nq, D)).astype(np.float64)
        if Nr >= 2:                                        # midpoints of two refs one step of 2 apart on one feature
            j = rng.integers(0, Nr, (B, Nq))
            qry = np.take_along_axis(ref, j[..., None], 1).copy()
            c = rng.integers(0, D, (B, Nq))
            bi, qi = np.meshgrid(np.arange(B), np.arange(Nq), indexing="ij")
            k = rng.integers(0, Nr, (B, Nq))
            ref[bi[:, :Nq // 2], k[:, :Nq // 2]] = qry[:, :Nq // 2]
            ref[bi[:, :Nq // 2], k[:, :Nq // 2], c[:, :Nq // 2]] += 2.0
            qry[bi, qi, c] += 1.0
        return ref.astype(F32), qry.astype(F32)
    ref = rng.standard_normal((B, Nr, D))
    qry = rng.standard_normal((B, Nq, D))
    if kind == "overflow":
        s = 1e19 / np.sqrt(D)                              # sum of D squared differences about 2e38: either side of 3.4e38
        ref = ref * s
        qry = qry * s
        qry[:, ::3] = 3e20 * np.sign(rng.standard_normal((B, len(qry[0, ::3]), D)))
        ref[:, ::2] = -np.abs(ref[:, ::2]) - 1e20
        return ref.astype(F32), qry.astype(F32)
    ref, qry = ref.astype(F32), qry.astype(F32)
    plant = []                                             # (query, ref row it must take)
    if Nr > 64:
        for j in range(min(3, Nr - 64)):                   # duplicates 64 apart: tiles j // 64 and j // 64 + 1
            ref[:, j + 64] = ref[:, j]
            plant.append(j)
        ref[:, Nr - 1] = ref[:, 5 % Nr]                    # and the last tile
        plant.append(5 % Nr)
    if D > 32 and Nr >= 8:                                 # rows 6 and 7 equal in features 0..31
        ref[:, 7, :32] = ref[:, 6, :32]
        ref[:, 6, 32:] = ref[:, 7, 32:] + F32(0.5)
        plant.append(7)
    if Nr >= 12:
        ref[:, 9] = np.nextafter(ref[:, 8], F32(np.inf))   # one ulp apart
        ref[:, 10] = 0.0
        plant += [9, 10]
    for i, j in enumerate(plant[:Nq]):
        qry[:, i] = ref[:, j]
    if kind == "offset":
        ref = (ref.astype(np.float64) + 1e4).astype(F32)
        qry = (qry.astype(np.float64) + 1e4).astype(F32)
    return ref, qry


def _knn_chunks(ref, qry, budget=1 << 24):
    """Yield (b0, b1, q0, q1, d32, d64): the squared distances [b1-b0, q1-q0, Nr] of a block of queries, in fp32 summed
    over the features in order from +0 (one rounding per operation, as the kernel: eager torch ops never fuse) and in
    float64."""
    B, Nq, D = qry.shape
    Nr = ref.shape[1]
    if Nq * Nr <= budget:
        gb, gq = max(1, budget // max(1, Nq * Nr)), Nq
    else:
        gb, gq = 1, max(1, budget // Nr)
    for b0 in range(0, B, gb):
        b1 = min(B, b0 + gb)
        r = ref[b0:b1]
        for q0 in range(0, Nq, gq):
            q1 = min(Nq, q0 + gq)
            q = qry[b0:b1, q0:q1]
            d32 = torch.zeros((b1 - b0, q1 - q0, Nr), dtype=torch.float32, device=ref.device)
            d64 = torch.zeros((b1 - b0, q1 - q0, Nr), dtype=torch.float64, device=ref.device)
            for c in range(D):
                t = q[:, :, None, c] - r[:, None, :, c]
                d32 = d32 + t * t
                t = q[:, :, None, c].double() - r[:, None, :, c].double()
                d64 = d64 + t * t
            yield b0, b1, q0, q1, d32, d64


def knn_fp32(ref, qry):
    """The literal fp32 restatement: (dist [B,Nq] f32, idx [B,Nq] int64), the first fp32 minimum and sqrtf of it.  The
    square root is taken in float64 and rounded once to fp32, which is the correctly rounded fp32 square root (53 >=
    2 * 24 + 2); torch's fp32 sqrt on the CPU is not correctly rounded everywhere."""
    ref, qry = _t(ref), _t(qry, _t(ref).device)
    B, Nq = qry.shape[:2]
    dist = torch.empty((B, Nq), dtype=torch.float32, device=ref.device)
    idx = torch.empty((B, Nq), dtype=torch.int64, device=ref.device)
    for b0, b1, q0, q1, d32, _ in _knn_chunks(ref, qry):
        i = torch.argmin(d32, -1)                          # the first minimal index (torch's documented tie rule)
        idx[b0:b1, q0:q1] = i
        dist[b0:b1, q0:q1] = torch.sqrt(d32.gather(-1, i[..., None])[..., 0].double()).float()
    return dist, idx


def _first_equal(rows):
    """[N] index of the first row bitwise equal to each row."""
    v = np.ascontiguousarray(rows.view(np.int32).reshape(len(rows), -1))
    _, first, inv = np.unique(v, axis=0, return_index=True, return_inverse=True)
    return first[inv.reshape(-1)]


def check_knn(ref, qry, dist, idx, literal=True):
    """bx_knn1's (dist, idx) [B,Nq] against the literal fp32 restatement (``literal``: bits equal) and float64 (the
    module docstring): decided arg-mins float64's first minimum, the others within the margin and never a later copy of
    an equal row, the distance within its bound of sqrt(d64).  Rows whose fp32 minimum is +inf: index 0, dist +inf."""
    ref, qry = _t(ref), _t(qry)
    qry = qry.to(ref.device)
    dist, idx = _t(dist).to(ref.device).reshape(qry.shape[:2]), _t(idx).to(ref.device).reshape(qry.shape[:2]).long()
    B, Nq, D = qry.shape
    Nr = ref.shape[1]
    out = dict(knn_queries=B * Nq, knn_undecided=0, knn_all_inf=0, knn_arg_ratio=0.0, knn_dist_ratio=0.0)
    assert bool(((idx >= 0) & (idx < Nr)).all()), "index outside [0, Nr)"
    if literal:
        d_l, i_l = knn_fp32(ref, qry)
        bad = (i_l != idx) | (d_l.view(torch.int32) != dist.view(torch.int32))
        assert not bool(bad.any()), f"differs from the literal fp32 arithmetic at {torch.nonzero(bad)[:5].tolist()}"
    ref_np = ref.cpu().numpy()
    first = np.stack([_first_equal(ref_np[b]) for b in range(B)]) if B * Nr else np.zeros((B, Nr), np.int64)
    idx_np = idx.cpu().numpy()
    assert (np.take_along_axis(first, idx_np, 1) == idx_np).all(), "a later copy of an equal ref row won a tie"
    kd = KN * (D + 3) / 2 + 1
    for b0, b1, q0, q1, d32, d64 in _knn_chunks(ref, qry):
        got = idx[b0:b1, q0:q1]
        inf = torch.isinf(d32.min(-1).values)
        out["knn_all_inf"] += int(inf.sum())
        if bool(inf.any()):
            assert bool((got[inf] == 0).all()) and bool(torch.isinf(dist[b0:b1, q0:q1][inf]).all()), \
                "all distances +inf: not (index 0, dist +inf)"
        keep = ~inf
        M = d64[keep].cpu().numpy()
        if len(M) == 0:
            continue
        two = torch.topk(d64[keep], min(2, Nr), -1, largest=False).values.cpu().numpy()
        best, second = two[:, 0], (two[:, 1] if Nr > 1 else np.full(len(two), np.inf))
        r, und = _nn_side(M, best, second, got[keep].cpu().numpy(), Nr, "knn", C=D)
        out["knn_arg_ratio"] = max(out["knn_arg_ratio"], r)
        out["knn_undecided"] += und
        s64 = np.sqrt(best)
        dk = dist[b0:b1, q0:q1][keep].cpu().numpy().astype(np.float64)
        bound = kd * U * s64 + 1e-15
        ratio = np.abs(dk - s64) / bound
        assert (ratio <= 1).all(), f"distance outside its bound of sqrt(d64): {ratio.max():.3g}"
        out["knn_dist_ratio"] = max(out["knn_dist_ratio"], float(ratio.max(initial=0.0)))
    return out


def check_radius_decision(dist, src, tgt, vs, D=3):
    """get_matching_indices' ``dist < search_voxel_size`` (the fp32 comparison) equals float64's ``sqrt(d64) < vs``
    wherever |sqrt(d64) - vs| exceeds the distance bound.  -> ratios and counts."""
    src, tgt = _t(src), _t(tgt)
    dist = _t(dist).to(src.device).reshape(-1).double()
    vs = float(F32(vs))
    best = torch.empty(src.shape[0], dtype=torch.float64, device=src.device)
    for _, _, q0, q1, _, d64 in _knn_chunks(tgt[None], src[None]):
        best[q0:q1] = d64[0].min(-1).values
    s64 = torch.sqrt(best)
    bound = (KN * (D + 3) / 2 + 1) * U * s64 + 1e-15
    dec = (s64 - vs).abs() > bound
    bad = dec & ((dist < vs) != (s64 < vs))
    assert not bool(bad.any()), f"dist < {vs} differs from float64 at {torch.nonzero(bad).flatten()[:5].tolist()}"
    return dict(vs_undecided=int((~dec).sum()), vs_matches=int((dist < vs).sum()))


# ------------------------------------------------------------------------------------------------ SVD
SVD_KINDS = ("random", "rank2", "rank1", "zero", "isotropic", "two_equal", "gap1e-7", "gap1e-5", "graded_cols",
             "graded_rows", "negdet", "signed_perm", "diag", "cov", "subnormal", "large")


def _rot(rng, n):
    q, r = np.linalg.qr(rng.standard_normal((n, 3, 3)))
    return q * np.sign(np.diagonal(r, axis1=1, axis2=2))[:, None, :]


def _signed_perms(rng, n):
    P = np.zeros((n, 3, 3))
    for k in range(n):
        P[k, np.arange(3), rng.permutation(3)] = rng.choice([-1.0, 1.0], 3)
    return P


def svd_case(kind, n=200, seed=0):
    """[n,3,3] fp32 matrices of one class of the catalogue (SVD_KINDS)."""
    rng = np.random.default_rng(seed)
    rnd = rng.standard_normal((n, 3, 3))
    sv = lambda s: _rot(rng, n) @ (np.asarray(s)[..., None] * _rot(rng, n).transpose(0, 2, 1))
    small = lambda shape: rng.integers(-4, 5, shape).astype(np.float64)
    if kind == "random":
        A = rnd
    elif kind == "rank2":
        A = np.einsum("ki,kj->kij", small((n, 3)), small((n, 3))) + np.einsum("ki,kj->kij", small((n, 3)), small((n, 3)))
    elif kind == "rank1":
        A = np.einsum("ki,kj->kij", small((n, 3)), small((n, 3)))
    elif kind == "zero":
        A = np.zeros((n, 3, 3))
    elif kind == "isotropic":                               # exact (signed permutations) and to rounding (rotations)
        c = rng.uniform(0.1, 10, (n, 1, 1))
        A = np.where(np.arange(n)[:, None, None] % 2 == 0, _signed_perms(rng, n), _rot(rng, n)) * c
    elif kind == "two_equal":
        s = rng.uniform(0.5, 2, n)
        A = sv(np.stack([s, s, s * rng.uniform(0, 0.9, n)], 1) * np.where(np.arange(n) % 2 == 0, 1, -1)[:, None])
        A[1::2] = sv(np.stack([s, s * 0.5, s * 0.5], 1))[1::2]
    elif kind in ("gap1e-7", "gap1e-5"):
        g = float(kind[3:])
        A = sv(np.stack([np.ones(n), np.full(n, 1 - g), np.full(n, 0.5)], 1))
        A[1::2] = sv(np.stack([np.ones(n), np.full(n, 0.5), np.full(n, 0.5 - 0.5 * g)], 1))[1::2]
    elif kind == "graded_cols":
        A = rnd * np.array([1.0, 1e-10, 1e-20])[None, None, :]
    elif kind == "graded_rows":
        A = rnd * np.array([1.0, 1e-10, 1e-20])[None, :, None]
    elif kind == "negdet":
        A = rnd.copy()
        A[np.linalg.det(A) > 0, :, 0] *= -1.0
    elif kind == "signed_perm":
        A = _signed_perms(rng, n) * rng.uniform(0.5, 2, (n, 1, 1))
    elif kind == "diag":
        d = rng.choice([0.0, 0.0, -1.0, 2.0, -3.5, 0.25], (n, 3))
        A = np.einsum("ki,ij->kij", d, np.eye(3))
    elif kind == "cov":                                     # cal_Z_axis: local = p - centre (the last point), local^T local
        A = np.empty((n, 3, 3))
        for k in range(n):
            off = (0.0, 10.0, 1e3, 1e4)[k % 4]
            p = rng.uniform(-0.3, 0.3, (512, 3)) * [1.0, 1.0, rng.choice([0.0, 1e-3, 3e-2])]
            p = (p @ _rot(rng, 1)[0].T + off).astype(F32)
            local = (p - p[-1]).astype(F32).astype(np.float64)
            A[k] = local.T @ local
    elif kind == "subnormal":
        A = rnd * 1e-40
    elif kind == "large":
        A = rnd * 1e30
    else:
        raise ValueError(kind)
    A = A.astype(F32)
    assert np.isfinite(A).all()
    return A


def _clusters(s, smax):
    """Split the descending s64 [3] into clusters: a gap above 2^10 KS u53 s_max separates them."""
    cl, cur = [], [0]
    for i in range(1, 3):
        if s[i - 1] - s[i] > 2.0 ** 10 * KS * U53 * smax:
            cl.append(cur)
            cur = []
        cur.append(i)
    return cl + [cur]


def check_svd(A, U_, S_, V_):
    """bx_svd3's (U, S, V) [B,3,3]/[B,3] on fp32 A [B,3,3] against numpy's float64 SVD: the bounds of the module
    docstring.  -> the largest ratio of each bound and the numbers of vectors and projectors checked."""
    host = lambda t: (t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)).astype(np.float64)
    A, Ug, S, Vg = host(A), host(U_), host(S_), host(V_)
    B = len(A)
    out = dict(svd_matrices=B, svd_vectors=0, svd_projectors=0)
    if B == 0:
        return out
    assert np.isfinite(Ug).all() and np.isfinite(S).all() and np.isfinite(Vg).all(), "non-finite output"
    assert (S[:, :-1] >= S[:, 1:]).all() and (S >= 0).all(), "S not descending and non-negative"
    u0, s0, vt0 = np.linalg.svd(A)
    v0 = vt0.transpose(0, 2, 1)
    smax = s0[:, :1]
    bS = U * s0 + (1 + U) * KS * U53 * smax + TINY
    out["S"] = float((np.abs(S - s0) / bS).max())
    assert out["S"] <= 1, f"S outside u s + KS u53 s_max: {out['S']:.3g} of the bound at {np.argmax((np.abs(S - s0) / bS).max(1))}"
    I = np.eye(3)
    for name, M in (("UtU", Ug), ("VtV", Vg)):
        e = np.abs(M.transpose(0, 2, 1) @ M - I).max((1, 2)) / (3 * U)
        out[name] = float(e.max())
        assert out[name] <= 1, f"{name}: |M^T M - I| {out[name]:.3g} of 3u at {int(np.argmax(e))}"
    nA = np.linalg.norm(A, axis=(1, 2))
    rec = np.linalg.norm(np.einsum("kij,kj,klj->kil", Ug, S, Vg) - A, axis=(1, 2))
    e = rec / ((3 * U + 4 * U * U + 2 * KS * U53) * nA + 2 * TINY)
    out["rec"] = float(e.max())
    assert out["rec"] <= 1, f"reconstruction {out['rec']:.3g} of its bound at {int(np.argmax(e))}"
    res = np.linalg.norm(np.einsum("kij,kjl->kil", A, Vg) - Ug * S[:, None, :], axis=1)
    e = res / (U * (smax + 2 * S + U * S) + 2 * KS * U53 * smax + 2 * TINY)
    out["pair"] = float(e.max())
    assert out["pair"] <= 1, f"||A v_i - s_i u_i|| {out['pair']:.3g} of its bound at {np.unravel_index(np.argmax(e), e.shape)}"
    vec, proj = 0.0, 0.0
    for k in range(B):
        if smax[k, 0] == 0:
            continue
        cl = _clusters(s0[k], smax[k, 0])
        for c in cl:
            rest = [j for j in range(3) if j not in c]
            g = min((abs(s0[k, i] - s0[k, j]) for i in c for j in rest), default=np.inf)
            w = KS * U53 * smax[k, 0] / g
            for got, want in ((Ug[k], u0[k]), (Vg[k], v0[k])):
                if len(c) == 1:
                    i = c[0]
                    err = min(np.abs(got[:, i] - want[:, i]).max(), np.abs(got[:, i] + want[:, i]).max())
                    r = err / (w + 2 * U)
                    assert r <= 1, f"matrix {k}: singular vector {i} {r:.3g} of its bound"
                    vec = max(vec, r)
                    out["svd_vectors"] += 1
                else:
                    Pg, Pw = got[:, c] @ got[:, c].T, want[:, c] @ want[:, c].T
                    r = np.abs(Pg - Pw).max() / (w + 3 * U)
                    assert r <= 1, f"matrix {k}: projector of cluster {c} {r:.3g} of its bound"
                    proj = max(proj, r)
                    out["svd_projectors"] += 1
    out["vec"], out["proj"] = float(vec), float(proj)
    return out


# ------------------------------------------------------------------------------------------------ gather / group
def gather_want(features, idx):
    """out[b,c,...] = features[b,c,idx[b,...]] bit for bit, NaN 0x7fc00000 where idx is outside [0, N): as int32 bits."""
    f = np.ascontiguousarray(features.cpu().numpy() if isinstance(features, torch.Tensor) else features, F32).view(np.int32)
    i = np.asarray(idx.cpu().numpy() if isinstance(idx, torch.Tensor) else idx).astype(np.int64)
    B, C, N = f.shape
    flat = i.reshape(B, 1, -1)
    ok = (flat >= 0) & (flat < N)
    g = np.take_along_axis(f, np.broadcast_to(np.where(ok, flat, 0), (B, C, flat.shape[2])), 2)
    g = np.where(np.broadcast_to(ok, g.shape), g, np.int32(NAN_BITS))
    return g.reshape((B, C) + i.shape[1:])


def check_gather(features, idx, out):
    got = np.ascontiguousarray(out.cpu().numpy() if isinstance(out, torch.Tensor) else out, F32).view(np.int32)
    want = gather_want(features, idx)
    assert got.shape == want.shape, f"shape {got.shape} != {want.shape}"
    bad = got != want
    assert not bad.any(), f"gather differs at {np.argwhere(bad)[:5].tolist()}"
    i = np.asarray(idx.cpu().numpy() if isinstance(idx, torch.Tensor) else idx)
    N = (features.shape[2])
    return dict(gather_elems=int(got.size), gather_out_of_range=int(((i < 0) | (i >= N)).sum()))
