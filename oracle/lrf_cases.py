"""Hand-built LRF patches at the edges of the covariance / eigenvector / Rodrigues chain (a4+a5), and the per-patch
float64 bounds the LRF is held to, for tests/test_lrf_fp64_*.py (the derivation of every bound is in the docstring of
tests/test_lrf_fp64_cpu.py).

TEST INFRASTRUCTURE ONLY.  ``lrf_patches(P, r)`` returns [K,P,3] fp32 patches, key point last, the other points within
about r of it, and one label per patch:
  * generic anisotropic patches, planes with random normals, poles (rank 1 plus noise), near-isotropic clouds;
  * exact and 1e-5-tilted horizontal planes below the sensor (c_z < 0: z -> +e_z) and above it (c_z > 0: z -> -e_z);
  * exactly collinear points (an axis-parallel line: rank 1 in fp32 exactly), an exact octahedron (isotropic);
  * all points equal to the key point (zero covariance), the empty-ball form (P - 1 copies of one point: rank 1);
  * key points at the origin and 1e-7 from it, coordinates offset by 1e3.
For P = 1 every patch is the key point alone and for P = 2 every covariance has rank 1: the cases then collapse into
those regimes, which is the point of running them."""
import numpy as np

from . import oracle as O

F32 = np.float32
U = 2.0 ** -24                 # fp32 unit roundoff

KZ = 8.0                       # z axis: angle <= KZ u lam_3 / gap
KS = 8.0                       # sign rule: decided by rounding when |z64 . c| <= (b_z + KS u) |c|_1
KR = 8.0                       # entries of R: rounding of the Rodrigues formula
KD = 8.0                       # delta: rounding of p - c, R x and / r
KO = 16.0                      # orthonormality of R
ANGULAR = 1e-2                 # b_z above this: z is only held to the near-null eigenspace
VACUOUS = 1e-2                 # an elementwise R bound above this is replaced by the invariants


def _rot(rng):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    return q


def _ball(rng, n, r):
    u = rng.normal(size=(n, 3))
    return u / np.linalg.norm(u, axis=1, keepdims=True) * r * rng.uniform(0, 1, (n, 1)) ** (1 / 3)


def _centre(rng, kind="generic"):
    if kind == "origin":
        return np.zeros(3)
    if kind == "near_origin":
        return rng.normal(size=3) * 1e-7
    if kind == "offset":
        return np.array([1e3, -1e3, 1e3]) + rng.uniform(-1, 1, 3)
    return rng.uniform(-3, 3, 3)


def lrf_patches(P, r=1.0, seed=0):
    """-> (patches [K,P,3] fp32, labels [K])."""
    rng = np.random.default_rng(seed)
    n = P - 1
    pats, labels = [], []

    def add(label, c, pts):
        c = np.asarray(c, np.float64).astype(F32)
        out = np.empty((P, 3), F32)
        out[:n] = np.asarray(pts, np.float64).reshape(n, 3).astype(F32)
        out[n] = c
        pats.append(out)
        labels.append(label)

    def aniso(c, sig):
        return c + (_ball(rng, n, r) * sig) @ _rot(rng).T

    for i in range(4):
        c = _centre(rng)
        add("anisotropic", c, aniso(c, (1.0, 0.5, 0.2)))
    for i in range(3):
        c = _centre(rng)
        add("anisotropic_mild", c, aniso(c, (1.0, 0.9, 0.7)))
    for i in range(4):                                                  # planes with random normals, no noise
        c = _centre(rng)
        add("plane", c, aniso(c, (1.0, 1.0, 0.0)))
    for cz in (-1.5, 1.5):
        c = np.array([rng.uniform(-2, 2), rng.uniform(-2, 2), cz])
        xy = _ball(rng, n, r)[:, :2]
        flat = np.concatenate([c[:2] + xy, np.full((n, 1), F32(cz))], axis=1)
        add("horizontal_below" if cz < 0 else "horizontal_above", c, flat)
        tilt = np.array([1.0, 0.3, 0.0]) * 1e-5
        tilted = np.concatenate([c[:2] + xy, (cz + xy @ tilt[:2])[:, None]], axis=1)
        add("tilted_below" if cz < 0 else "tilted_above", c, tilted)
    for i in range(3):                                                  # poles: rank 1 plus noise
        c = _centre(rng)
        u = rng.normal(size=3)
        u /= np.linalg.norm(u)
        add("pole", c, c + np.outer(rng.uniform(-r, r, n), u) + 1e-4 * r * rng.normal(size=(n, 3)))
    c = _centre(rng)
    line = np.repeat(c[None].astype(F32), n, axis=0).astype(np.float64)
    line[:, 0] = (F32(c[0]) + rng.uniform(-r, r, n)).astype(F32)
    add("collinear_axis", c, line)
    c = _centre(rng)
    u = rng.normal(size=3)
    add("collinear", c, c + np.outer(rng.uniform(-r, r, n), u / np.linalg.norm(u)))
    for i in range(2):
        c = _centre(rng)
        add("isotropic_ball", c, c + _ball(rng, n, r))
    c = np.round(_centre(rng), 2).astype(F32)
    octa = np.concatenate([np.eye(3), -np.eye(3)]) * F32(r)
    oc = c.astype(np.float64) + octa[np.arange(n) % 6]
    add("octahedron", c, oc)
    add("octahedron_perturbed", c, oc + 1e-4 * r * rng.normal(size=oc.shape))
    c = _centre(rng)
    add("all_equal", c, np.repeat(c[None], n, axis=0))
    q = c + r * 0.5 * rng.normal(size=3)
    add("empty_ball", c, np.repeat(q[None], n, axis=0))
    for kind in ("origin", "near_origin", "offset"):
        for sig in ((1.0, 0.5, 0.2), (1.0, 1.0, 0.0)):
            c = _centre(rng, kind)
            add(f"{kind}_{'plane' if sig[2] == 0 else 'anisotropic'}", c, aniso(c, sig))
    return np.stack(pats), np.array(labels)


def report(name, out):
    """Print the largest ratios and the branch counts of check_lrf results (run pytest with -s)."""
    ratios = {k: v for k, v in out.items() if isinstance(v, float)}
    counts = {k: v for k, v in out.items() if isinstance(v, int)}
    print(f"\n[lrf-fp64] {name}: " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items())
          + (" | " + ", ".join(f"{k} {v}" for k, v in counts.items()) if counts else ""))


def merge(acc, out):
    """Fold one check_lrf result into acc: ratios by maximum, counts by sum."""
    for k, v in out.items():
        acc[k] = max(acc.get(k, 0.0), v) if isinstance(v, float) else acc.get(k, 0) + v
    return acc


# ------------------------------------------------------------------------------------------------ bounds
def _round_out32(v, up):
    """The fp32 value nearest to v on the far side (>= v if up, else <= v)."""
    f = np.asarray(v, np.float64).astype(F32)
    bad = (f.astype(np.float64) < v) if up else (f.astype(np.float64) > v)
    f[bad] = np.nextafter(f[bad], F32(np.inf) if up else F32(-np.inf))
    return f.astype(np.float64)


def angle(a, b):
    """Unsigned angle between the lines of a and b [K,3] (atan2 of |a x b| and |a . b| on normalised vectors)."""
    a = a / np.linalg.norm(a, axis=1, keepdims=True)
    b = b / np.linalg.norm(b, axis=1, keepdims=True)
    return np.arctan2(np.linalg.norm(np.cross(a, b), axis=1), np.abs(np.einsum("ki,ki->k", a, b)))


def check_lrf(patches, des_r, aligned, stable, delta, Rt, ra, z=None):
    """Hold one LRF output (delta [K,P,3], Rt [K,3,3], rand_axis [K,3], fp32) to ``oracle.lrf_fp64`` patch by patch.
    ``z`` [K,3]: the fp32 z axes themselves (the oracle's ``want_z``); without it z is the third column of Rt, which in
    the literal form carries the acos error of theta as well.  Asserts every bound; returns the largest ratio of each
    check (err / bound) and the number of patches that took each branch."""
    patches = np.asarray(patches, F32)
    K, P, _ = patches.shape
    delta, Rt, ra = (np.asarray(a, np.float64) for a in (delta, Rt, ra))
    ref = O.lrf_fp64(patches, des_r, aligned, stable)
    r = np.broadcast_to(np.asarray(des_r, F32).astype(np.float64), (K,))
    pt = patches.astype(np.float64)
    c = pt[:, -1]
    x = pt - c[:, None]
    out = {}
    assert np.isfinite(delta).all() and np.isfinite(Rt).all() and np.isfinite(ra).all(), "non-finite output"
    if aligned:
        assert (Rt == np.eye(3)).all(), "aligned: R is not I"
        assert (ra == (1.0, 0.0, 0.0)).all(), "aligned: rand_axis is not e_x"
        want = x / r[:, None, None]
        ulp = np.spacing(np.abs(want).astype(F32)).astype(np.float64)
        err = np.abs(delta - want)
        assert (err <= 2 * ulp).all(), f"aligned: delta beyond 2 ulps at {np.argwhere(err > 2 * ulp)[:3].tolist()}"
        out["delta_ulps"] = float((err / np.maximum(ulp, 1e-45)).max(initial=0))
        return out
    R = Rt.transpose(0, 2, 1)                                  # the rotation applied to delta
    lam, gap, C = ref["lam"], ref["gap"], ref["C"]
    l3 = lam[:, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        b_z = np.where(gap > 0, KZ * U * l3 / gap, np.inf)
    ang_ok = b_z <= ANGULAR
    z64 = ref["z"]
    # a zero axis (rand_axis[:2] == 0) means the kernel's fp32 z had z_0 = z_1 = 0 exactly: z = +-e_z, R = I.  (z_0 / 1e-12
    # cannot underflow to 0 for a non-zero fp32 z_0.)  Read from R alone, the line of that z is known (e_z) but not its
    # sign; the line is held to float64's below like every other z, so a zero axis on a patch whose float64 z is not
    # vertical fails the z check.
    deg = (ra[:, 0] == 0) & (ra[:, 1] == 0)
    if z is None:
        zk = Rt[:, :, 2].copy()
        zk[deg] = (0.0, 0.0, 1.0)
        signed = ~deg
    else:
        zk = np.asarray(z, np.float64)
        signed = np.ones(K, bool)
        assert (zk[deg, :2] == 0).all(), f"zero axis for a z off the vertical at patches {np.flatnonzero(deg & (zk[:, :2] != 0).any(axis=1))[:5].tolist()}"
    # sign rule: must equal the float64 one unless |z64 . c| is within the z bound and the rounding of the fp32 sum
    s = np.sign(np.einsum("ki,ki->k", zk, z64))
    s[(s == 0) | ~signed] = 1.0
    with np.errstate(invalid="ignore"):
        clear = ang_ok & signed & (ref["margin"] > (b_z + KS * U) * np.abs(c).sum(axis=1))
    flips = clear & (s < 0)
    assert not flips.any(), f"sign rule differs from float64 on {int(flips.sum())} patches, first {np.flatnonzero(flips)[:5].tolist()}"
    out["sign_checked"], out["sign_by_rounding"] = int(clear.sum()), int((ang_ok & ~clear).sum())
    zr = z64 * s[:, None]                                     # the float64 axis on the kernel's side where rounding decides
    Rr, rar = O.rodrigues_fp64(zr, stable)
    cz, sn = zr[:, 2], np.hypot(zr[:, 0], zr[:, 1])
    # theta: the float64 angle against the fp32 cosines the kernel can see
    with np.errstate(invalid="ignore"):
        eps_c = np.minimum(b_z * sn + 0.5 * b_z * b_z, 2.0) + KR * U
    if stable:
        dth = np.minimum(b_z, np.pi) + KR * U
    else:
        th = np.arccos(np.clip(cz, -1, 1))
        lo = _round_out32(np.clip(cz - eps_c, -1, 1), up=False)
        hi = _round_out32(np.clip(cz + eps_c, -1, 1), up=True)
        dth = np.maximum(np.abs(np.arccos(np.clip(lo, -1, 1)) - th), np.abs(np.arccos(np.clip(hi, -1, 1)) - th)) + 2 * np.pi * U
    with np.errstate(divide="ignore", invalid="ignore"):
        da = np.where(sn > 0, np.minimum(2.0, 2.0 * (b_z + KR * U) / sn), 2.0)
    # z: an angle where the spectrum separates the smallest eigenvalue, else the near-null eigenspace.  Read from the
    # literal form's R, z carries theta's acos error too -- except at a zero axis, where it is e_z exactly.
    extra = np.zeros(K) if (stable or z is not None) else np.where(deg, 0.0, dth)
    zt = b_z + extra
    a = angle(zk, z64)
    g = ang_ok
    if g.any():
        rz = a[g] / zt[g]
        assert (rz <= 1).all(), f"z angle beyond bound: worst ratio {rz.max():.3g} at patch {np.flatnonzero(g)[np.argmax(rz)]}"
        out["z"] = float(rz.max())
    wide = ~ang_ok
    if wide.any():
        zn = zk[wide] / np.linalg.norm(zk[wide], axis=1, keepdims=True)
        excess = np.maximum(np.linalg.norm(np.einsum("kij,kj->ki", C[wide], zn), axis=1) - lam[wide, 0], 0.0)
        tol = KZ * U * l3[wide] + l3[wide] * np.minimum(extra[wide], 2.0)
        with np.errstate(divide="ignore", invalid="ignore"):
            rr = np.where(tol > 0, excess / tol, np.where(excess > 0, np.inf, 0.0))
        assert (rr <= 1).all(), f"z outside the near-null eigenspace: worst ratio {rr.max():.3g}"
        out["z_eigenspace"] = float(rr.max())
    out["z_angular"], out["z_eigenspace_n"] = int(g.sum()), int(wide.sum())
    assert (Rt[deg] == np.eye(3)).all(), "R != I where the axis is zero"
    tiny = ang_ok & (sn < 1e-12)
    assert deg[tiny].all(), f"sn < 1e-12 without R = I at patches {np.flatnonzero(tiny & ~deg)[:5].tolist()}"
    out["R_identity"] = int(deg.sum())
    # R elementwise where the bound means something, else the invariants
    bR = dth + (2.0 * (1.0 - cz) + sn) * da + KR * U
    elem = ang_ok & (bR <= VACUOUS) & ~deg
    if elem.any():
        e = np.abs(R[elem] - Rr[elem]).max(axis=(1, 2)) / bR[elem]
        assert (e <= 1).all(), f"R beyond bound: worst ratio {e.max():.3g} at patch {np.flatnonzero(elem)[np.argmax(e)]}"
        out["R"] = float(e.max())
        xl1 = np.abs(x[elem]).sum(axis=2, keepdims=True)
        want = np.einsum("kij,kpj->kpi", Rr[elem], x[elem]) / r[elem, None, None]
        tol = (bR[elem, None, None] + KD * U) * xl1 / r[elem, None, None]
        with np.errstate(divide="ignore", invalid="ignore"):
            e = np.where(tol > 0, np.abs(delta[elem] - want) / tol, 0.0)
        assert (e <= 1).all(), f"delta against R64 beyond bound: worst ratio {e.max():.3g}"
        out["delta_vs_R64"] = float(e.max())
    inv = ~elem & ~deg
    if inv.any():
        I3 = np.eye(3)
        o = np.abs(np.einsum("kij,klj->kil", R[inv], R[inv]) - I3).max(axis=(1, 2)) / (KO * U)
        assert (o <= 1).all(), f"R not orthonormal: worst ratio {o.max():.3g}"
        dt = np.abs(np.linalg.det(R[inv]) - 1.0) / (KO * U)
        assert (dt <= 1).all(), f"det R != 1: worst ratio {dt.max():.3g}"
        out["R_orthonormal"] = float(max(o.max(), dt.max()))
        g = inv & ang_ok
        if g.any():
            e = np.linalg.norm(np.einsum("kij,kj->ki", R[g], zr[g]) - (0.0, 0.0, 1.0), axis=1) / (b_z[g] + dth[g] + KR * U)
            assert (e <= 1).all(), f"|R z64 - e_z| beyond bound: worst ratio {e.max():.3g}"
            out["Rz"] = float(e.max())
    out["R_elementwise_n"], out["R_invariants_n"] = int(elem.sum()), int(inv.sum())
    # rand_axis: the axis (z_1, -z_0) / sn
    g = ang_ok & ~deg & (da < 2)
    if g.any():
        e = np.abs(ra[g] - rar[g]).max(axis=1) / da[g]
        assert (e <= 1).all(), f"rand_axis beyond bound: worst ratio {e.max():.3g}"
        out["rand_axis"] = float(e.max())
    assert (ra[:, 2] == 0).all()
    # delta against the kernel's own R applied in float64
    want = np.einsum("kij,kpj->kpi", R, x) / r[:, None, None]
    tol = KD * U * np.einsum("kij,kpj->kpi", np.abs(R), np.abs(x)) / r[:, None, None]
    err = np.abs(delta - want)
    with np.errstate(divide="ignore", invalid="ignore"):
        e = np.where(tol > 0, err / tol, np.where(err > 0, np.inf, 0.0))
    assert (e <= 1).all(), f"delta against its own R beyond bound: worst ratio {e.max():.3g}"
    out["delta_own_R"] = float(e.max(initial=0))
    return out
