"""Hand-built SPT patches at the edges of the voxel ball query (a6), for tests/test_descnet_fp64_*.py.

TEST INFRASTRUCTURE ONLY.  ``spt_patches`` returns [K,P,3] fp32 patches mixing:
  * points at fp32 squared distance exactly r^2 from a voxel centre (where one exists on the walk) or the last one outside,
    and the point one ulp inside;
  * points on the z axis (planar radius 0), with +-0.0 in x and y;
  * points at azimuth 0, just below 2 pi, and on the bin edges j * 2 pi / azi_n;
  * points on a ring of the table (planar radius and z of a (shell, elevation) row: d_r = 0);
  * points outside the unit ball (up to |p| = 1.5), points with -0.0 components;
  * clusters of 24 points around a voxel centre (more than nv and more than 16 hits in one ball);
  * exact-zero points (the key-point copies that pad a patch) interleaved with the others;
and the special patches: all zero; non-zero point 0 inside a ball; zero point 0 (the slot-0 rule)."""
import math

import numpy as np

from . import oracle as O

F32 = np.float32


def d2_f32(q, p):
    """The ball test's squared distance in the oracle's fp32 order ((dx^2 + dy^2) + dz^2), q [3] against p [n,3]."""
    q, p = np.asarray(q, F32), np.asarray(p, F32)
    dx, dy, dz = q[0] - p[:, 0], q[1] - p[:, 1], q[2] - p[:, 2]
    return (dx * dx + dy * dy) + dz * dz


def rows(vox, azi_n):
    """(planar radius, z) of every (shell, elevation) row, computed like the kernel (fp32)."""
    c = vox[::azi_n]
    return np.sqrt(c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1]), c[:, 2].copy()


def boundary_pair(c, u, rho):
    """Two points on the line from voxel centre c along u at distance ~rho: the first with d2 >= r^2 (== where the ulp walk
    meets it) and its neighbour one ulp further in (d2 < r^2).  None if the walk does not straddle r^2."""
    r2 = F32(rho) * F32(rho)
    p0 = (c.astype(np.float64) + rho * u).astype(F32)
    i = int(np.argmax(np.abs(u)))
    towards = F32(c[i])
    cand = [p0[i]]
    for direction in (towards, F32(np.sign(p0[i] - c[i]) * 10.0 + p0[i])):
        v = p0[i]
        for _ in range(48):
            v = np.nextafter(v, direction, dtype=F32)
            cand.append(v)
    cand = np.unique(np.asarray(cand, F32))
    pts = np.repeat(p0[None], len(cand), axis=0)
    pts[:, i] = cand
    d2 = d2_f32(c, pts)
    inside, outside = d2 < r2, d2 >= r2
    if not inside.any() or not outside.any():
        return None
    return pts[outside][np.argmin(d2[outside])], pts[inside][np.argmax(d2[inside])]


def edge_points(vox, rho, azi_n, rng):
    """The pool of non-special points (fp32 [n,3])."""
    Rc, cz = rows(vox, azi_n)
    step = 2 * math.pi / azi_n
    pts = []
    for v in rng.choice(len(vox), min(len(vox), 40), replace=False):
        u = rng.normal(size=3)
        u /= np.linalg.norm(u)
        bp = boundary_pair(vox[v], u, rho)
        if bp is not None:
            pts += list(bp)
        for ax in range(3):                                      # along an axis: d2 == r^2 is reachable exactly
            e = np.zeros(3)
            e[ax] = 1.0
            bp = boundary_pair(vox[v], e, rho)
            if bp is not None:
                pts += list(bp)
    for z in np.linspace(-1.2, 1.2, 13):                         # the z axis
        pts += [(0.0, 0.0, z), (-0.0, 0.0, z), (0.0, -0.0, z)]
    for r in range(len(Rc)):
        R, z = float(Rc[r]), float(cz[r])
        pts += [(R, 0.0, z), (0.0, R, z), (-R, 0.0, z), (0.0, -R, z), (R, -0.0, z)]    # on the ring, d_r = 0
        pts += [(R * math.cos(t), R * math.sin(t), z) for t in rng.uniform(0, 2 * math.pi, 2)]
        for j in range(azi_n):                                   # bin edges, at the ring and off it
            rr = R if j % 2 else 0.5 * R + 0.1
            pts.append((rr * math.cos(j * step), rr * math.sin(j * step), z))
        pts += [(R, -R * 1e-7, z), (R, -1e-30, z), (0.3, float(np.nextafter(F32(0), F32(-1))), z)]   # just below 2 pi
    for _ in range(40):                                          # outside the unit ball
        u = rng.normal(size=3)
        pts.append(u / np.linalg.norm(u) * rng.uniform(1.0, 1.5))
    for _ in range(20):                                          # -0.0 components
        p = rng.uniform(-0.8, 0.8, 3)
        p[rng.integers(0, 3)] = -0.0
        pts.append(p)
    u = rng.normal(size=(120, 3))
    pts += list(u / np.linalg.norm(u, axis=1, keepdims=True) * rng.uniform(0, 1, (120, 1)) ** (1 / 3))
    pts = np.asarray(pts, dtype=np.float64).astype(F32)
    return pts[rng.permutation(len(pts))]


def cluster(vox, rng, n=24):
    c = vox[rng.integers(0, len(vox))]
    return (c + 1e-3 * rng.normal(size=(n, 3))).astype(F32)


def spt_patches(P, rad_n=3, azi_n=20, ele_n=7, rho=0.8 / 3, seed=0):
    """[K,P,3] fp32: patch 0 all zero; 1: non-zero point 0 on a voxel centre; 2: zero point 0; 3: clusters; the rest drawn
    from the edge pool, with exact zeros interleaved.  K grows for small P so that the whole pool is visited."""
    rng = np.random.default_rng(seed)
    vox = O.voxel_table(rad_n, azi_n, ele_n)
    pool = edge_points(vox, rho, azi_n, rng)
    K = int(min(64, max(8, math.ceil(len(pool) / P))))
    out = np.zeros((K, P, 3), F32)
    o = 0

    def draw(n):
        nonlocal o
        idx = (o + np.arange(n)) % len(pool)
        o += n
        return pool[idx]

    for k in range(1, K):
        p = draw(P)
        if k == 3 or k % 4 == 0:
            cl = np.concatenate([cluster(vox, rng) for _ in range(3)])[:P]
            p[rng.choice(P, len(cl), replace=False)] = cl
        if k != 1 and P > 1:
            p[rng.random(P) < 0.3] = 0.0                          # exact-zero padding, interleaved
        if k == 1:
            p[0] = vox[rng.integers(0, len(vox))]
        if k == 2:
            p[0] = 0.0
        out[k] = p
    return out
