"""Edge inputs for the training-stage kernels (csrc/bx_train.cu: ground-truth matches, SO(2) augmentation, EquiMatch, the
SO(2) label) and the float64 checks they are held to, shared by tests/test_train_fp64_*.py (the derivation of every
bound is in the docstring of tests/test_train_fp64_cpu.py).

TEST INFRASTRUCTURE ONLY.  The builders return fp32 inputs; the ``check_*`` functions take the inputs and what an
implementation returned (the fp32 oracle of oracle/train_stages.py, a kernel, or torch on CUDA), assert the bounds
against the float64 restatements of oracle/train_stages.py and return the largest ratio (err / bound) of each check and
the number of decisions left to rounding (``merge`` / ``report`` as in oracle/pose_cases.py)."""
import numpy as np
import torch

from . import train_stages as TS
from .pose_cases import merge  # noqa: F401  (re-exported for the tests)

F32 = np.float32
U = 2.0 ** -24                 # fp32 unit roundoff

KQ = 5.0                       # transform: |fl(q_j) - q_j| <= KQ u (sum_k |R_jk| |p_k| + |t_j|)
KD = 4.0                       # distance from an fp32 q: |fl(d) - d| <= KD u d
KS = 4.0                       # sin / cos / acos: 2 ulp, i.e. <= 4 u |value|
KM = 4.0                       # one 3-term dot product: |err| <= KM u sum |a_k| |b_k|
KL = 4.0                       # label arithmetic: angle * azi_n / fp32(2 pi), fp32(2 pi) itself, 2 pi - angle

GT_M = (0, 1, 2047, 2048, 2049, 4097)
GT_N = (0, 1, 127, 129, 1023, 1024, 1025, 5000)
OFFSETS = (1e2, 1e3, 1e4)
VOXEL = 0.05


def report(name, out):
    ratios = {k: v for k, v in out.items() if isinstance(v, float)}
    counts = {k: v for k, v in out.items() if isinstance(v, int)}
    print(f"\n[train-fp64] {name}: " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items())
          + (" | " + ", ".join(f"{k} {v}" for k, v in counts.items()) if counts else ""))


def _rot(rng):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q))


def _pose(rng, offset=0.0):
    T = np.eye(4)
    T[:3, :3] = _rot(rng)
    T[:3, 3] = rng.uniform(-1, 1, 3) + np.array([1.0, -0.5, 0.25]) * offset / np.sqrt(1.3125)
    return T.astype(F32)


# ------------------------------------------------------------------------------------------------ ground-truth matches
def gt_case(N, M, seed=0, offset=0.0, dup=False, voxel=VOXEL):
    """-> (src [N,3], tgt [M,3], T [4,4], voxel) fp32: targets in a 2 m cube (at ``offset`` m from the origin), about two
    thirds of the sources a target pulled back through T^-1 with noise of the order of the voxel, the rest anywhere.
    ``dup``: the second half of the targets repeats the first bit for bit."""
    rng = np.random.default_rng(seed)
    T = _pose(rng, offset)
    c = T[:3, 3].astype(np.float64)
    tgt = (c + rng.uniform(-1, 1, (M, 3))).astype(F32)
    if dup and M >= 2:
        tgt[(M + 1) // 2:] = tgt[:M // 2]
    T64 = T.astype(np.float64)
    near = rng.random(N) < 0.67
    x = c + rng.uniform(-1.2, 1.2, (N, 3))
    if M:
        x[near] = tgt[rng.integers(0, M, int(near.sum()))] + rng.normal(scale=voxel * 0.6, size=(int(near.sum()), 3))
    src = ((x - T64[:3, 3]) @ T64[:3, :3]).astype(F32)
    return src, tgt, T, voxel


def gt_voxel_edge_case(voxel=VOXEL):
    """Identity pose; targets on the integer grid (i, j, 0), sources at (i, j, +-s) with s the fp32 voxel, one fp32 ulp
    below and above it.  Every fp32 operation is exact here (dz = s, sqrt(fl(s * s)) = s), so the distance is s in fp32
    and in float64: -> (src, tgt, T, voxel, expected keep [N] of the strict test)."""
    v = F32(voxel)
    ss = np.array([v, np.nextafter(v, F32(0)), np.nextafter(v, F32(1))], F32)
    g = np.stack(np.meshgrid(np.arange(-4, 5), np.arange(-4, 5), indexing="ij"), -1).reshape(-1, 2).astype(F32)
    tgt = np.concatenate([g, np.zeros((len(g), 1), F32)], 1)
    src, keep = [], []
    for k, (i, j) in enumerate(g):
        s = ss[k % 3] * (1 if k % 2 else -1)
        src.append((i, j, s))
        keep.append(k % 3 == 1)
    return np.asarray(src, F32), tgt, np.eye(4, dtype=F32), float(v), np.asarray(keep)


def gt_cases():
    """name -> (src, tgt, T, voxel) of every synthetic case (C1 / C2 come from add_training_clouds)."""
    out = {}
    for M in GT_M:
        for N in GT_N:
            out[f"M{M}_N{N}"] = gt_case(N, M, seed=M * 7 + N)
    out["dup"] = gt_case(5000, 4097, seed=1, dup=True)
    for o in OFFSETS:
        out[f"offset{o:g}"] = gt_case(3000, 2049, seed=int(o), offset=o)
    src, tgt, T, v, _ = gt_voxel_edge_case()
    out["voxel_edge"] = (src, tgt, T, v)
    return out


def training_pair(name, seed=0):
    """The second-level clouds add_training_clouds builds for the C1 / C2 pair -> (src, tgt, T, voxel)."""
    from bufferx_b200.synth import add_training_clouds, make_pair, workload_cfg
    cfg = workload_cfg(name)
    d = add_training_clouds(make_pair(name, seed), cfg)
    return d["src_sds_pcd"], d["tgt_sds_pcd"], np.asarray(d["relt_pose"], F32), float(np.asarray(d["voxel_sizes"]).reshape(-1)[0])


def check_gt(src, tgt, T, voxel, pairs, rows=None):
    """pairs [C,2] ([i, nn(i)] as returned, C the count) against matching_indices_fp64 on the source rows ``rows``
    (default all).  Per row the distance margin is m(d) = |e_q| + KD u d (e_q the transform's error); the arg-min is decided
    where second - best > m(best) + m(second) and must then be float64's, an undecided pick lies within m of the minimum,
    and among bitwise-equal targets the first index wins.  Keep / drop equals float64's wherever |d - voxel| > m(d) (d the
    float64 distance of the pick; a dropped row's minimum).  Pairs are in source order; with every row checked the count
    lies in [decided kept, decided kept + marginal]."""
    src, tgt = np.asarray(src, F32).reshape(-1, 3), np.asarray(tgt, F32).reshape(-1, 3)
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    N, M = len(src), len(tgt)
    if M == 0 or N == 0:
        assert len(pairs) == 0, "matches without a source or a target point"
        return dict(rows=0)
    assert (np.diff(pairs[:, 0]) > 0).all() and (pairs[:, 0] >= 0).all() and (pairs[:, 0] < N).all(), "pairs not in source order"
    assert ((pairs[:, 1] >= 0) & (pairs[:, 1] < M)).all(), "target index out of range"
    rows = np.arange(N) if rows is None else np.asarray(rows)
    ref = TS.matching_indices_fp64(src, tgt, T, voxel, rows=rows)
    eq = KQ * U * np.linalg.norm(ref["qmag"], axis=1)
    marg = lambda d, e=eq: e + KD * U * d + 1e-14 * (1 + d)
    kept = np.full(N, -1, np.int64)
    kept[pairs[:, 0]] = pairs[:, 1]
    got = kept[rows]
    k = got >= 0
    dec = (ref["second"] - ref["best"]) > marg(ref["best"]) + marg(ref["second"])
    bad = k & dec & (got != ref["arg"])
    assert not bad.any(), f"decided arg-min differs at rows {rows[bad][:5].tolist()}"
    q = ref["q"][k]
    dg = np.sqrt(((q - tgt[got[k]].astype(np.float64)) ** 2).sum(1))
    pick = (dg - ref["best"][k]) / (marg(ref["best"][k], eq[k]) + marg(dg, eq[k]))
    assert (pick <= 1).all(), f"pick outside the margin of the minimum at rows {rows[k][pick > 1][:5].tolist()}"
    key = tgt.view(np.int32)
    uniq, inv = np.unique(key, axis=0, return_inverse=True)
    first = np.full(len(uniq), M, np.int64)
    np.minimum.at(first, inv.reshape(-1), np.arange(M))
    assert (first[inv.reshape(-1)[got[k]]] == got[k]).all(), "a later copy of a bitwise-equal target won a tie"
    v = ref["voxel"]
    bad_keep = dg >= v + marg(dg, eq[k])
    assert not bad_keep.any(), f"kept beyond the voxel at rows {rows[k][bad_keep][:5].tolist()}"
    drop = ~k
    bad_drop = drop & (ref["best"] < v - marg(ref["best"]))
    assert not bad_drop.any(), f"dropped a decided match at rows {rows[bad_drop][:5].tolist()}"
    marginal = np.abs(ref["best"] - v) <= marg(ref["best"])
    out = dict(rows=int(len(rows)), argmin_undecided=int((~dec).sum()), keep_marginal=int(marginal.sum()),
               pick=float(np.maximum(pick, 0).max(initial=0.0)))
    if len(rows) == N:
        lo = int((ref["keep"] & ~marginal).sum())
        assert lo <= len(pairs) <= lo + int(marginal.sum()), f"count {len(pairs)} outside [{lo}, {lo + int(marginal.sum())}]"
    return out


# ------------------------------------------------------------------------------------------------ SO(2) augmentation
AUG_P = (1, 255, 256, 257, 1024)
AUG_K = (0, 1, 700)


def threshold_angles():
    """fp32 angles within a few ulps of fp32(1e-3), on both sides of kornia's theta^2 > fp32(1e-6), with both signs."""
    a = F32(1e-3)
    out = [a]
    lo = hi = a
    for _ in range(6):
        lo, hi = np.nextafter(lo, F32(0)), np.nextafter(hi, F32(1))
        out += [lo, hi]
    out = np.asarray(out, F32)
    return np.concatenate([out, -out])


def edge_angles():
    two_pi_below = np.nextafter(F32(2 * np.pi), F32(0))
    while float(two_pi_below) >= 2 * np.pi:
        two_pi_below = np.nextafter(two_pi_below, F32(0))
    return np.concatenate([np.asarray([0.0, 1e-4, -1e-4, np.pi / 2, np.pi, 3 * np.pi / 2, two_pi_below], F32),
                           threshold_angles()])


def aug_case(K, P, seed=0):
    """-> (delta [K,P,3], rand_axis [K,3], angles [K]) fp32: the reference's draw, the edge angles first."""
    rng = np.random.RandomState(seed)
    delta = rng.uniform(-1, 1, size=(K, P, 3)).astype(F32)
    ra = rng.normal(size=(K, 3)).astype(F32)
    ang = TS.draw_aug_angles(rng, K)
    e = edge_angles()
    ang[:min(K, len(e))] = e[:K]
    return delta, ra, ang


def aug_R_bound(a):
    """Elementwise bound [K,3,3] on an fp32 evaluation of the full kornia form at the fp32 angles a against float64:
    th = sqrtf(fl(a a)) within 1.5 u th; sinf / cosf within KS u of their value plus |d sin| <= |cos| dth; the axis
    a / (th + 1e-6) within 1.5 u th / (th + 1e-6) + 2 u; products and the last sum one u each."""
    a = np.asarray(a, F32).astype(np.float64)
    th = np.abs(a)
    e = TS.AUG_THRESHOLD
    c, s = np.cos(th), np.sin(th)
    wz = a / (th + e)
    dth = 1.5 * U * th
    ec = np.abs(s) * dth + KS * U * np.abs(c)
    es = np.abs(c) * dth + KS * U * np.abs(s)
    rwz = 1.5 * U * th / (th + e) + 2 * U
    ews = np.abs(wz * s) * (rwz + U) + np.abs(wz) * es
    r22 = c + wz * wz * (1 - c)
    e22 = ec * np.abs(1 - wz * wz) + np.abs(1 - c) * (2 * rwz + 4 * U) + U * np.abs(r22)
    z = np.zeros_like(a)
    return 2 * np.stack([ec, ews, z, ews, ec, z, z, z, e22], axis=1).reshape(-1, 3, 3)


def check_aug(delta_in, ra_in, angles, delta_out, ra_out, aug_R):
    """The rotations and rotated rows of one so2_augment call against so2_augment_fp64.  R elementwise within
    aug_R_bound (the first-order form is exact: 1, +-a, 0); where the branch is undecided either branch's matrix.  Rows
    within KM u |R| |d| + |dR| |d| of float64 (|dR| the bound of the accepted branch).  aug_R is the R that was applied:
    the rows are bit for bit the fixed-order fp32 product with the returned aug_R."""
    delta_in, ra_in = np.asarray(delta_in, F32), np.asarray(ra_in, F32)
    K = len(angles)
    if K == 0:
        return dict(patches=0)
    ref = TS.so2_augment_fp64(delta_in, ra_in, angles)
    R = np.asarray(aug_R, F32).reshape(K, 3, 3).astype(np.float64)
    bf = aug_R_bound(angles)
    tiny = 1e-300
    r_full = (np.abs(R - ref["R_full"]) / (bf + tiny)).reshape(K, -1).max(1)
    ok_taylor = (R == ref["R_taylor"]).reshape(K, -1).all(1)
    full_ok = r_full <= 1
    want_full = ref["full"]
    okk = np.where(ref["decided"], np.where(want_full, full_ok, ok_taylor), full_ok | ok_taylor)
    assert okk.all(), (f"R off at patches {np.flatnonzero(~okk)[:5].tolist()} (angles {np.asarray(angles)[~okk][:3].tolist()}, "
                       f"ratio to the full form {r_full[~okk][:3].tolist()})")
    used_full = np.where(ok_taylor, False, True)
    bR = np.where(used_full[:, None, None], bf, 0.0)
    R64 = np.where(used_full[:, None, None], ref["R_full"], ref["R_taylor"])
    out = dict(patches=K, branch_undecided=int((~ref["decided"]).sum()), R=float(np.where(used_full, r_full, 0).max()))
    for what, din, dout in (("rows", delta_in.reshape(K, -1, 3), np.asarray(delta_out, F32).reshape(K, -1, 3)),
                            ("rand_axis", ra_in.reshape(K, 1, 3), np.asarray(ra_out, F32).reshape(K, 1, 3))):
        d = din.astype(np.float64)
        exp = np.einsum("kpj,kij->kpi", d, R64)
        bound = KM * U * np.einsum("kpj,kij->kpi", np.abs(d), np.abs(R)) + np.einsum("kpj,kij->kpi", np.abs(d), bR) + 1e-300
        r = np.abs(dout - exp) / bound
        assert (r <= 1).all(), f"{what}: {r.max():.3g} of the bound at patch {int(np.argmax(r.reshape(K, -1).max(1)))}"
        out[what] = float(r.max())
        same = TS._rotate_rows(din, np.asarray(aug_R, F32).reshape(K, 1, 3, 3)).astype(F32)
        assert np.array_equal(same, dout), f"{what}: not the fixed-order product with the returned aug_R"
    return out


# ------------------------------------------------------------------------------------------------ EquiMatch
EQ_C = (1, 31, 32, 33, 64)
EQ_K = (1, 5, 7)
EQ_L = (1, 2, 20, 32)
EQ_LIMIT = 6144                # 2 C K L floats <= 48 KB of shared memory


def equi_case(B, C, K, L, kind="unit", seed=0):
    """-> (d1, d2) [B,C,K,L] fp32: "unit" maps normalised over C with d2 a noisy roll of d1 (a clear arg-max),
    "raw" unnormalised maps of magnitude up to 1e3, "cancel" pairs of channels whose products cancel to a few ulps."""
    g = torch.Generator().manual_seed(seed)
    d1 = torch.randn(B, C, K, L, generator=g)
    if kind == "raw":
        d1 = d1 * torch.exp(3 * torch.rand(B, C, 1, 1, generator=g) * 2.3)
        d2 = torch.randn(B, C, K, L, generator=g) * 10
    else:
        d1 = torch.nn.functional.normalize(d1, dim=1)
        d2 = torch.nn.functional.normalize(d1 + 0.5 * torch.randn(B, C, K, L, generator=g), dim=1)
        d2 = torch.roll(d2, shifts=min(5, L - 1), dims=-1)
    if kind == "cancel" and C >= 2:
        h = C // 2
        d1[:, h:2 * h] = d1[:, :h]
        d2[:, h:2 * h] = -d2[:, :h] * (1 + 1e-6 * torch.randn(B, h, K, L, generator=g))
    return d1.float().contiguous(), d2.float().contiguous()


def equi_terms_kernel(C, K, L):
    """Rounding steps of one bx_equi_match score: one lane's sequential sum of ceil(C/32) K L products, then the 5-level
    xor tree."""
    return -(-C // 32) * K * L + 5


def check_equi(d1, d2, got, n_terms, chunk_elems=2 ** 24):
    """|got - ref64| <= gamma_n sum |d1| |d2| (per score), and the arg-max over shifts equals float64's where the top gap
    exceeds twice the row's largest bound (eqv_acc is that arg-max)."""
    d1, d2 = torch.as_tensor(d1).float(), torch.as_tensor(d2).float()
    got = np.asarray(got, np.float64)
    B, C, K, L = d1.shape
    if B == 0:
        return dict(rows=0)
    ref, mag = np.empty((B, L)), np.empty((B, L))
    step = max(1, chunk_elems // (C * K * L * L))
    for a in range(0, B, step):
        x1, x2 = d1[a:a + step].double(), d2[a:a + step].double()
        ref[a:a + step] = TS.equi_match(x1, x2).numpy()
        mag[a:a + step] = TS.equi_match(x1.abs(), x2.abs()).numpy()
    g = n_terms * U / (1 - n_terms * U)
    bound = g * mag + 1e-300
    r = np.abs(got - ref) / bound
    assert (r <= 1).all(), f"score error {r.max():.3g} of gamma_{n_terms} sum|d1||d2| at row {int(np.argmax(r.max(1)))}"
    srt = np.sort(ref, axis=1)
    gap = srt[:, -1] - (srt[:, -2] if L > 1 else -np.inf)
    dec = gap > 2 * bound.max(1)
    bad = dec & (got.argmax(1) != ref.argmax(1))
    assert not bad.any(), f"decided arg-max differs at rows {np.flatnonzero(bad)[:5].tolist()}"
    return dict(rows=B, argmax_undecided=int((~dec).sum()), score=float(r.max()))


# ------------------------------------------------------------------------------------------------ SO(2) label
GT_AZI = (1, 4, 20, 36)
GT_P = (0, 1, 129, 4000)


def _rotations(rng, n):
    return np.stack([_rot(rng) for _ in range(n)]).astype(F32) if n else np.zeros((0, 3, 3), F32)


def _rz(b):
    c, s = np.cos(b), np.sin(b)
    z, o = np.zeros_like(b), np.ones_like(b)
    return np.stack([c, -s, z, s, c, z, z, z, o], -1).reshape(-1, 3, 3)


def label_case(kind, P=4000, azi_n=20, seed=0):
    """-> (s_rand_axis [P,3], s_R [P,3,3], t_R [P,3,3], T [4,4], aug_R [P,3,3] or None) fp32.
    "random" / "aug": random unit axes, frames and pose (with the reference's augmentation draw).  "axis": the target
    axis exactly +-z (the fp32 projection is 0), and 1e-4 and 1e-7 off it.  "align": u = (cos a, sin a, 0) and v = u rotated
    about z by beta, with beta = 0 (theta = 0), pi (theta = pi), labels k + 1/2 +- a few ulps and beta just below 2 pi."""
    rng = np.random.default_rng(seed)
    eye = np.broadcast_to(np.eye(3, dtype=F32), (P, 3, 3)).copy()
    if kind in ("random", "aug"):
        ra = rng.normal(size=(P, 3))
        ra /= np.linalg.norm(ra, axis=1, keepdims=True)
        T = np.eye(4, dtype=F32)
        T[:3, :3] = _rot(rng)
        T[:3, 3] = [0.3, -0.2, 0.1]
        A = TS.aug_rotations(TS.draw_aug_angles(np.random.RandomState(seed), P)) if kind == "aug" else None
        return ra.astype(F32), _rotations(rng, P), _rotations(rng, P), T, A
    if kind == "axis":
        off = np.array([0.0, 1e-4, 1e-7])[np.arange(P) % 3]
        sign = np.where(np.arange(P) % 2, 1.0, -1.0)
        phi = rng.uniform(0, 2 * np.pi, P)
        v = np.stack([off * np.cos(phi), off * np.sin(phi), sign * np.sqrt(1 - off ** 2)], 1)
        ra = rng.normal(size=(P, 3))
        ra /= np.linalg.norm(ra, axis=1, keepdims=True)
        # t_R maps ra (T = I) onto v: t_R = Q with ra @ Q = v, Q = rotation taking ra to v (Rodrigues)
        tR = np.asarray([_align(ra[i], v[i]) for i in range(P)], F32).reshape(P, 3, 3)
        ra32 = ra.astype(F32)
        exact = off == 0
        # exact +-z: s = e_z, t_R = +-I, so v = (0, 0, +-1) in fp32 without rounding
        ra32[exact] = [0, 0, 1]
        tR[exact] = eye[exact] * sign[exact, None, None].astype(F32)
        return ra32, _rotations(rng, P), tR, np.eye(4, dtype=F32), None
    if kind == "align":
        alpha = rng.uniform(0, 2 * np.pi, P)
        ra = np.stack([np.cos(alpha), np.sin(alpha), np.zeros(P)], 1)
        k = rng.integers(0, azi_n, P)
        j = np.arange(P) % 11 - 5
        beta = (k + 0.5) * 2 * np.pi / azi_n + j * 4 * U * 2 * np.pi
        beta[0::13] = 0.0
        beta[1::13] = np.pi
        beta[2::13] = 2 * np.pi - 1e-7 * (1 + np.arange(len(beta[2::13])) % 5)
        beta[3::13] = 2 * np.pi - 1e-6
        # v = ra @ t_R = ra rotated by beta about z: t_R = Rz(beta)^T
        tR = np.swapaxes(_rz(beta), 1, 2)
        return ra.astype(F32), eye, tR.astype(F32), np.eye(4, dtype=F32), None
    raise ValueError(kind)


def _align(a, b):
    """A rotation Q with a @ Q = b (unit a, b)."""
    v = np.cross(a, b)
    c = float(a @ b)
    if np.linalg.norm(v) < 1e-12:
        return np.eye(3) if c > 0 else -np.eye(3) + 2 * np.outer(_perp(a), _perp(a))
    K = np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])
    M = np.eye(3) + K + K @ K / (1 + c)        # M a = b
    return M.T


def _perp(a):
    p = np.cross(a, [1.0, 0, 0] if abs(a[0]) < 0.9 else [0, 1.0, 0])
    return p / np.linalg.norm(p)


def _abs_dot(a, B, transpose=False):
    return np.einsum("pk,pjk->pj" if transpose else "pk,pkj->pj", np.abs(a), np.abs(B))


def label_bound(s_ra, s_R, t_R, T, azi_n, aug_R=None):
    """so2_gt_fp64 and the error bound of an fp32 evaluation of it -> (ref, e_lab, defined, sign_decided, zero_proj).
    Vectors: each 3-term product within KM u sum |a||b| plus the propagated input error, giving e_u and e_v.  The unit
    projection moves by dp <= |e_vxy| / (|v_xy| - |e_vxy|) + 4 u; the cosine by d_cs <= dp + 2 |e_u| / |u| + 10 u; the
    angle by min(d_cs / sqrt(1 - (|cs| + d_cs)^2), (pi / sqrt 2) sqrt(d_cs)) plus acosf (KS u pi) and KL u 2 pi for
    2 pi - angle and fp32(2 pi).  e_lab = azi_n / 2 pi of that plus KL u azi_n.  Undefined where |v_xy| <= 2 |e_vxy|.
    The sign is decided where |cz| > |u_xy| dp + |e_u_xy| + 4 u (|u0 p1| + |u1 p0|)."""
    f = lambda x: np.asarray(x, F32).astype(np.float64)
    ref = TS.so2_gt_fp64(s_ra, s_R, t_R, T, azi_n, aug_R)
    s = f(s_ra).reshape(-1, 3)
    G = np.broadcast_to(f(T)[:3, :3].T, (len(s), 3, 3))
    e_t = KM * U * _abs_dot(s, G)
    e_u = KM * U * _abs_dot(s, f(s_R).reshape(-1, 3, 3))
    B = np.abs(f(t_R).reshape(-1, 3, 3))
    e_v = np.einsum("pk,pkj->pj", e_t, B) + KM * U * _abs_dot(ref["t"], B)
    if aug_R is not None:
        A = np.abs(f(aug_R).reshape(-1, 3, 3))
        e_v = np.einsum("pk,pjk->pj", e_v, A) + KM * U * _abs_dot(ref["v_pre_aug"], A, transpose=True)
    exy = np.hypot(e_v[:, 0], e_v[:, 1])
    vxy = ref["vxy"]
    defined = vxy > 2 * exy
    dp = np.where(defined, exy / np.maximum(vxy - exy, 1e-300), 2.0) + 4 * U
    unorm = ref["unorm"]
    dcs = dp + 2 * np.linalg.norm(e_u, axis=1) / unorm + 10 * U
    top = np.abs(ref["cs"]) + dcs
    lin = np.where(top < 1, dcs / np.sqrt(np.maximum(1 - top * top, 1e-300)), np.inf)
    dth = np.minimum(lin, np.pi / np.sqrt(2) * np.sqrt(dcs)) + KS * U * np.pi + KL * U * 2 * np.pi
    e_lab = azi_n / (2 * np.pi) * dth + KL * U * azi_n
    u = ref["u"]
    e_cz = np.hypot(u[:, 0], u[:, 1]) * dp + np.hypot(e_u[:, 0], e_u[:, 1]) \
        + 4 * U * (np.abs(u[:, 0] * ref["p"][:, 1]) + np.abs(u[:, 1] * ref["p"][:, 0]))
    sign_dec = np.abs(ref["cz"]) > e_cz
    # the kernel's own fp32 projection, in its order (bit-identical with -fmad=false): exactly 0 gives the reference's
    # value cos = 0, theta = pi / 2
    s32 = np.asarray(s_ra, F32).reshape(-1, 3)
    T32 = np.asarray(T, F32)
    t32 = np.stack([((s32[:, 0] * T32[j, 0]) + (s32[:, 1] * T32[j, 1])) + (s32[:, 2] * T32[j, 2]) for j in range(3)], 1)
    B32 = np.asarray(t_R, F32).reshape(-1, 3, 3)
    v32 = np.stack([((t32[:, 0] * B32[:, 0, j]) + (t32[:, 1] * B32[:, 1, j])) + (t32[:, 2] * B32[:, 2, j]) for j in range(3)], 1)
    if aug_R is not None:
        v32 = TS._rotate_rows(v32, np.asarray(aug_R, F32).reshape(-1, 3, 3)).astype(F32)
    zero = (v32[:, 0] == 0) & (v32[:, 1] == 0)
    return ref, e_lab, defined & ~zero, sign_dec, zero


def _round_half_even_wrap(x, azi_n):
    r = np.round(x)                  # numpy rounds half to even, like torch.round
    return np.where(r == azi_n, 0, r).astype(np.int64)


def check_label(s_ra, s_R, t_R, T, azi_n, got, integer, aug_R=None):
    """Labels of one so2_gt call.  All in [0, azi_n) and finite.  Float labels within e_lab of float64's, circularly
    (0 == azi_n); where the sign is undecided also the mirror azi_n - lab is accepted.  Integer labels equal float64's
    rounding wherever the label is more than e_lab from a half-integer (both mirrors where the sign is undecided).  Where
    |v_xy| is below its error bound the label is only required to be finite and in range, and where the fp32 projection is
    exactly 0, the reference's value azi_n / 4 (within KL u azi_n)."""
    got = np.asarray(got)
    P = len(got)
    if P == 0:
        return dict(labels=0)
    assert np.isfinite(got).all() and (got >= 0).all() and (got < azi_n).all(), \
        f"labels outside [0, {azi_n}): {got[(got < 0) | (got >= azi_n) | ~np.isfinite(got)][:5].tolist()}"
    ref, e_lab, defined, sign_dec, zero = label_bound(s_ra, s_R, t_R, T, azi_n, aug_R)
    lab, mir = ref["lab"], np.mod(azi_n - ref["lab"], azi_n)
    out = dict(labels=P, undefined=int((~defined).sum()), sign_undecided=int((defined & ~sign_dec).sum()))
    if integer:
        assert got.dtype == np.int64
        want = _round_half_even_wrap(lab, azi_n)
        want_m = _round_half_even_wrap(mir, azi_n)
        dec = defined & (ref["half"] > e_lab) & (sign_dec | ((np.abs(np.mod(mir, 1.0) - 0.5) > e_lab) & (want == want_m)))
        ok = (got == want) | (~sign_dec & (got == want_m))
        bad = dec & ~ok
        assert not bad.any(), f"decided integer labels differ at {np.flatnonzero(bad)[:5].tolist()}: {got[bad][:5].tolist()} vs {want[bad][:5].tolist()}"
        if zero.any():
            assert (got[zero] == _round_half_even_wrap(np.full(int(zero.sum()), azi_n / 4), azi_n)).all(), "zero projection: not round(azi_n / 4)"
        out["int_undecided"] = int((defined & ~dec).sum())
        out["int_near_half"] = float((e_lab / np.maximum(ref["half"], 1e-300))[dec].max(initial=0.0))
        return out
    g = got.astype(np.float64)
    circ = lambda x: np.minimum(np.abs(g - x), azi_n - np.abs(g - x))
    err = np.where(sign_dec, circ(lab), np.minimum(circ(lab), circ(mir)))
    r = err / e_lab
    bad = defined & (r > 1)
    assert not bad.any(), f"float labels beyond the bound at {np.flatnonzero(bad)[:5].tolist()}: {g[bad][:3].tolist()} vs {lab[bad][:3].tolist()}"
    if zero.any():
        assert (np.abs(g[zero] - azi_n / 4) <= KL * U * azi_n).all(), f"zero projection: {g[zero][:3].tolist()} not azi_n / 4"
    out["float"] = float(r[defined].max(initial=0.0))
    out["float_worst_err"] = float(err[defined].max(initial=0.0))
    return out
