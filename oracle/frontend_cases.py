"""Edge inputs and float64 checks of FPS, radius estimation and patch gathering (a1-a3), shared by
tests/test_frontend_fp64_cpu.py (the C oracle) and tests/test_frontend_fp64_gpu.py (the kernels).

Every check takes what a kernel (or the oracle) returned and holds it to the float64 evaluations of oracle.py
(fps_fp64, radius_count_bounds / radius_fp64 / radius_replay, ball_query_fp64, select_patches_fp64); the bounds are
derived in the docstring of tests/test_frontend_fp64_cpu.py.  Each returns a dict of ratios (floats, the largest is
kept by ``merge``) and counts (ints, summed), printed by ``report``."""
import functools

import numpy as np
import torch

from oracle import oracle as O
from oracle.pose_cases import merge  # noqa: F401  (re-exported for the tests)

U = O.U24
F32 = np.float32


def report(name, out):
    ratios = {k: v for k, v in out.items() if isinstance(v, float)}
    counts = {k: v for k, v in out.items() if isinstance(v, (int, np.integer))}
    print(f"\n[frontend-fp64] {name}: " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items())
          + (" | " + ", ".join(f"{k} {v}" for k, v in counts.items()) if counts else ""))


# ------------------------------------------------------------------------------------------------ a1
MAG_HI = F32(1e-3)                            # 1e-3f is the fp32 value just above the double 1e-3
MAG_LO = np.nextafter(F32(1e-3), F32(0))      # ... and this the one just below
assert float(MAG_LO) < 1e-3 < float(MAG_HI)


@functools.lru_cache(maxsize=None)
def _mag_exact_point(target):
    """(a, b, c) multiples of 2^-18 with a^2 + b^2 + c^2 == target exactly and every fp32 product and partial sum
    exact."""
    t = int(round(float(target) * 2.0 ** 36))
    assert t / 2.0 ** 36 == float(target)
    ex = lambda v: int(F32(v)) == v
    for a in range(int(t ** 0.5), 0, -1):
        rest = t - a * a
        if not ex(a * a):
            continue
        for b in range(min(a, int(rest ** 0.5)), -1, -1):
            c2 = rest - b * b
            c = int(round(c2 ** 0.5))
            if c * c == c2 and ex(b * b) and ex(c2) and ex(a * a + b * b):
                return np.array([a, b, c], np.float64) / 2.0 ** 18
    # none (1e-3f - ulp): a point whose fp32 magnitude rounds to the target (undecided in float64)
    rng = np.random.default_rng(7)
    while True:
        v = rng.normal(size=3)
        p = (v / np.linalg.norm(v) * np.sqrt(float(target))).astype(F32)
        if ((p[0] * p[0]) + (p[1] * p[1])) + (p[2] * p[2]) == target:
            return p.astype(np.float64)


def fps_cloud(kind, n, seed=0, offset=0.0, k_valid=3):
    """Edge clouds of FPS: 'uniform', 'dup' (every point four times), 'lattice' (integer grid: exact distance ties),
    'allskip' (every |p|^2 <= 1e-3), 'fewvalid' (all but k_valid inside the skip zone), 'magedge' (points with
    |p|^2 exactly the fp32 values either side of 1e-3), plus a translation ``offset`` along (1, 1, 1)."""
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        x = rng.uniform(-2, 2, (n, 3))
    elif kind == "dup":
        x = np.repeat(rng.uniform(-2, 2, ((n + 3) // 4, 3)), 4, axis=0)[:n]
        x = x[rng.permutation(n)]
    elif kind == "lattice":
        s = int(np.ceil(n ** (1 / 3)))
        g = np.stack(np.meshgrid(*[np.arange(s)] * 3, indexing="ij"), -1).reshape(-1, 3)[:n]
        x = g[rng.permutation(len(g))] * 0.25
    elif kind in ("allskip", "fewvalid"):
        x = rng.normal(size=(n, 3))
        x *= (rng.uniform(0, 0.03, n) / np.linalg.norm(x, axis=1))[:, None]
        if kind == "fewvalid":
            x[rng.choice(n, min(k_valid, n), replace=False)] = rng.uniform(0.2, 1.0, (min(k_valid, n), 3))
    elif kind == "magedge":
        x = rng.uniform(-1, 1, (n, 3))
        hi, lo = _mag_exact_point(MAG_HI), _mag_exact_point(MAG_LO)
        x[0], x[n // 3] = lo, hi
        x[1::7] = hi * rng.choice([-1, 1], (len(x[1::7]), 3))
        x[2::7] = lo * rng.choice([-1, 1], (len(x[2::7]), 3))
    else:
        raise ValueError(kind)
    return (x + offset).astype(F32)


FPS_KINDS = ("uniform", "dup", "lattice", "allskip", "fewvalid", "magedge")


def check_fps(xyz, npoint, idx, kpts=None):
    """idx[0] = 0; every pick a candidate (or index 0 when no point survives the skip); its float64 running minimum
    within kd*u*vmax of the largest; decided steps take float64's arg-max (any of the tied values); kpts = xyz[idx]."""
    host = lambda a: a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    idx = host(idx).reshape(-1)
    assert len(idx) == npoint
    if npoint == 0:
        return dict(fps_steps=0)
    assert idx[0] == 0 and (idx >= 0).all() and (idx < len(xyz)).all()
    if kpts is not None:
        assert np.array_equal(host(kpts).reshape(-1, 3), host(xyz)[idx]), "kpts != xyz[idx]"
    r = O.fps_fp64(xyz, idx)
    if npoint == 1:
        return dict(fps_steps=0)
    vmax, vpick, vsec = r["vmax"], r["vpick"], r["vsecond"]
    ok = r["pick_ok"]
    none = (torch.as_tensor(idx[1:]) == 0).to(ok.device) & (r["n_valid"] == 0)
    assert bool(ok.all()), f"FPS picked a skipped point at steps {torch.nonzero(~ok).flatten()[:8].tolist()}"
    gap = torch.where(none, torch.zeros_like(vmax), vmax - vpick)
    marg = 12.0 * U * vmax.clamp_min(0)
    bad = gap > marg
    assert not bool(bad.any()), f"FPS pick outside the margin at steps {torch.nonzero(bad).flatten()[:8].tolist()}"
    dec = r["decided"]
    wrong = dec & (gap > 0)
    assert not bool(wrong.any()), f"decided FPS step not float64's arg-max: {torch.nonzero(wrong).flatten()[:8].tolist()}"
    ratio = float((gap / marg.clamp_min(1e-300)).max())
    if r["n_valid"] == 0:
        assert (idx == 0).all(), "a cloud with every point skipped must pick index 0 at every step"
    return dict(fps_gap_ratio=ratio, fps_steps=npoint - 1, fps_undecided=int((~dec).sum()),
                fps_undecided_skip=r["n_undecided_skip"])


# ------------------------------------------------------------------------------------------------ a2
RADIUS_THRESHOLDS = (5.0, 2.0, 0.5)


def radius_case(kind, n=3000, kr=64, seed=0):
    """(kpts, pts) of a radius estimation: 'uniform' (a 6 m box), 'far' (every point beyond 5 m of every key point),
    'coincident' (key points drawn from the cloud), 'axis' (key points at the origin and points at r_m, r_m +- one step
    of 2^-13 along the axes: every pair exact, many on a threshold), 'd25' (points at d2 == 25 exactly, key points at
    the origin), 'off100' / 'off1000' (the uniform box at that offset, the norms' cancellation dominates), 'dense'
    (a 2 cm ball of points: the 0.5 % radius rounds to 0.0)."""
    rng = np.random.default_rng(seed)
    if kind in ("uniform", "off100", "off1000", "coincident"):
        off = {"off100": 100.0, "off1000": 1000.0}.get(kind, 0.0)
        pts = rng.uniform(-3, 3, (n, 3)) + off
        kp = pts[rng.choice(n, kr, replace=False)] if kind == "coincident" else rng.uniform(-3, 3, (kr, 3)) + off
    elif kind == "far":
        kp = rng.uniform(-1, 1, (kr, 3))
        v = rng.normal(size=(n, 3))
        pts = v / np.linalg.norm(v, axis=1, keepdims=True) * rng.uniform(7.0, 9.0, (n, 1))
    elif kind == "axis":
        kp = np.zeros((kr, 3))
        m = rng.integers(1, 400, n)
        r = 5.0 * m / 8192 + rng.choice([-1, 0, 0, 1], n) * 2.0 ** -13
        pts = np.zeros((n, 3))
        pts[np.arange(n), rng.integers(0, 3, n)] = r * rng.choice([-1, 1], n)
    elif kind == "d25":
        kp = np.zeros((kr, 3))
        pts = rng.uniform(-1, 1, (n, 3))
        e = np.array([[5.0, 0, 0], [0, -5.0, 0], [0, 0, 5.0], [3.0, 4.0, 0], [0, -3.0, 4.0]])
        pts[: n // 3] = e[rng.integers(0, 5, n // 3)]
    elif kind == "dense":
        v = rng.normal(size=(n, 3))
        pts = v / np.linalg.norm(v, axis=1, keepdims=True) * rng.uniform(0, 0.02, (n, 1))
        kp = pts[rng.choice(n, kr, replace=False)]
    else:
        raise ValueError(kind)
    return kp.astype(F32), pts.astype(F32)


RADIUS_KINDS = ("uniform", "far", "coincident", "axis", "d25", "off100", "off1000", "dense")


def check_radius_hist(cum, lo, hi):
    """lo[m] <= cum[m] <= hi[m] for every m (cum: the kernel's cumulative histogram, 8193 entries)."""
    cum = np.asarray(cum, np.int64)[:O.RADIUS_BINS + 1]
    bad = np.nonzero((cum < lo) | (cum > hi))[0]
    assert len(bad) == 0, f"histogram outside the float64 interval at m={bad[:8].tolist()}: {cum[bad[:4]]} vs {lo[bad[:4]]}..{hi[bad[:4]]}"
    w = hi - lo
    return dict(hist_undecided_bins=int((w > 0).sum()), hist_width_max=int(w.max()))


def check_radius(cum, denom, thresholds, tolerance, m_out, r_out, lo, hi):
    """Per threshold: the kernel's m reachable through the undecided decisions (equal when none), its radius
    float32(round(5 m / 8192, 2)), and the literal reference loop on the kernel's own cumulative histogram giving the
    same m and radius."""
    out = check_radius_hist(cum, lo, hi)
    und = 0
    for i, th in enumerate(thresholds):
        reach, u, radii = O.radius_fp64(lo, hi, denom, th, tolerance)
        m = int(m_out[i])
        assert m in reach, f"threshold {th}: m={m} not reachable, float64 allows {sorted(reach)[:8]}"
        if u == 0:
            assert reach == {m}
        assert F32(r_out[i]) == radii[m], f"threshold {th}: radius {r_out[i]} != {radii[m]}"
        rm, rr = O.radius_replay(cum, denom, th, tolerance)
        assert (rm, rr) == (m, F32(r_out[i])), f"threshold {th}: reference loop on the kernel's histogram gives {(rm, rr)}"
        und += u
    out["bisect_undecided"] = und
    return out


# ------------------------------------------------------------------------------------------------ a3
def cell_edge(r):
    return float(F32(F32(r) * F32(1.001)))


def patch_case(kind, n=3000, k=48, r=0.3, P=16, seed=0, offset=0.0):
    """(pts, kpts, r) of a patch gathering: 'uniform' (2 m box), 'exact' (points at fp32 distance exactly r from a
    key point, and one ulp inside), 'cells' (key points and points on cell boundaries, multiples of r*1.001 around 0),
    'counts' (balls with exactly P-1, P and P+1 hits in a sparse cloud), 'empty' (balls without points), 'big' (a
    radius larger than the cloud); ``offset`` translates everything."""
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        pts = rng.uniform(-1, 1, (n, 3))
        kp = pts[rng.choice(n, k, replace=False)] + rng.normal(scale=0.01, size=(k, 3))
    elif kind == "exact":
        r = 0.25
        kp = (np.round(rng.uniform(-1, 1, (k, 3)) * 64) / 64 + offset).astype(F32)
        pts = (rng.uniform(-1.5, 1.5, (n, 3)) + offset).astype(F32)
        h = n // 2
        ax = rng.integers(0, 3, h)
        base = kp[rng.integers(0, k, h)].copy()
        on = base[np.arange(h), ax] + F32(r) * rng.choice([-1, 1], h).astype(F32)        # exact: fp32 distance r
        inside = rng.random(h) < 0.5
        on[inside] = np.nextafter(on[inside], base[np.arange(h), ax][inside])             # one ulp inside
        base[np.arange(h), ax] = on
        pts[:h] = base
        return pts, kp, float(r)
    elif kind == "cells":
        c = cell_edge(r)
        g = rng.integers(-6, 7, (n, 3)) * c
        pts = g + rng.choice([0.0, 0.0, 1e-7, -1e-7], (n, 3))
        kp = rng.integers(-5, 6, (k, 3)) * c
    elif kind == "counts":
        kp = rng.uniform(-20, 20, (k, 3))
        blocks = []
        for j in range(k):
            h = (P - 1, P, P + 1)[j % 3]
            v = rng.normal(size=(h, 3))
            blocks.append(kp[j] + v / np.linalg.norm(v, axis=1, keepdims=True) * rng.uniform(0, 0.8 * r, (h, 1)))
        pts = np.concatenate(blocks + [rng.uniform(-20, 20, (max(n - sum(map(len, blocks)), 1), 3)) * 10 + 400])
        pts = pts[rng.permutation(len(pts))]
    elif kind == "empty":
        pts = rng.uniform(-1, 1, (n, 3))
        kp = rng.uniform(5, 6, (k, 3))
    elif kind == "big":
        pts = rng.uniform(-1, 1, (n, 3))
        kp = pts[rng.choice(n, k, replace=False)]
        r = 10.0
    else:
        raise ValueError(kind)
    return (pts + offset).astype(F32), (kp + offset).astype(F32), float(r)


PATCH_KINDS = ("uniform", "exact", "cells", "counts", "empty", "big")


def check_ball_query(xyz, qry, radius, idx, chunk=1 << 24):
    """Each row: strictly increasing listed prefix of hits or undecided points; no decided hit skipped below the last
    listed entry; when fewer than P are listed, no decided hit missing; the rest padded with the first index; an empty
    ball all zeros.  Batched form: xyz [B,N,3], qry [B,Q,3], idx [B,Q,P], every cloud's rows to its own points."""
    idx = torch.as_tensor(np.asarray(idx) if not isinstance(idx, torch.Tensor) else idx).long()
    q = qry if isinstance(qry, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(qry))
    p = xyz if isinstance(xyz, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(xyz))
    dev = p.device
    idx = idx.to(dev)
    if p.dim() == 3:
        out = {}
        step = max(1, chunk // max(1, q.shape[1] * p.shape[1]))
        for b in range(0, p.shape[0], step):
            merge(out, _check_ball_query_rows(lambda a, s: O.ball_query_fp64(p[b:b + step], q[b:b + step], radius).reshape(-1, p.shape[1]),
                                              idx[b:b + step].reshape(-1, idx.shape[-1]), p.shape[1], 1 << 62))
        return out
    return _check_ball_query_rows(lambda a, s: O.ball_query_fp64(p, q[a:a + s], radius), idx, p.shape[0], chunk)


def _check_ball_query_rows(status, idx, N, chunk):
    """check_ball_query on index rows [Q,P] whose float64 statuses [rows, N] status(a, step) gives for rows a..a+step."""
    dev = idx.device
    Q, P = idx.shape
    out = dict(bq_rows=Q, bq_undecided_pairs=0, bq_undecided_listed=0, bq_empty=0, bq_full=0)
    step = max(1, chunk // N)
    ar = torch.arange(N, device=dev)
    for a in range(0, Q, step):
        st = status(a, step)
        row = idx[a:a + step]
        inc = row[:, 1:] > row[:, :-1]
        c = 1 + torch.cumprod(inc.to(torch.int64), 1).sum(1)
        empty = (row == 0).all(1) & (st[:, 0] == 0)
        c = torch.where(empty, torch.zeros_like(c), c)
        slot = torch.arange(P, device=dev)[None, :]
        listed_slot = slot < c[:, None]
        s_at = st.gather(1, row)
        assert not bool(((s_at == 0) & listed_slot).any()), "a decided miss is listed"
        # listed points (padding slots scatter into a spare column N, so no False overwrites a listed index)
        L = torch.zeros((st.shape[0], N + 1), dtype=torch.bool, device=dev)
        L.scatter_(1, torch.where(listed_slot, row, torch.full_like(row, N)), True)
        L = L[:, :N]
        last = row.gather(1, (c - 1).clamp_min(0)[:, None])[:, 0]
        below = ar[None, :] < torch.where(c > 0, last, torch.full_like(last, -1))[:, None]
        skipped = (st == 1) & ~L & (below | (c < P)[:, None])
        assert not bool(skipped.any()), f"decided hit skipped in rows {(a + torch.nonzero(skipped.any(1)).flatten()[:8]).tolist()}"
        pad = torch.where(empty[:, None], torch.zeros_like(row), row[:, :1].expand(-1, P))
        assert bool(((row == pad) | listed_slot).all()), "padding is not the first index (all zeros for an empty ball)"
        out["bq_undecided_pairs"] += int((st == 2).sum())
        out["bq_undecided_listed"] += int(((s_at == 2) & listed_slot).sum())
        out["bq_empty"] += int(empty.sum())
        out["bq_full"] += int((c == P).sum())
    return out


def check_patches(pts_perm, kpts, idx, patches):
    """Patches equal the float64 mask formula of patch_embedder.py:105-111 applied to the index row, exactly."""
    want = O.select_patches_fp64(pts_perm, kpts, idx)
    got = patches if isinstance(patches, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(patches))
    got = got.to(want.device).to(torch.float64).reshape(want.shape)
    bad = got != want
    assert not bool(bad.any()), f"patch differs from the mask formula in rows {torch.nonzero(bad.any(2).any(1)).flatten()[:8].tolist()}"
    return dict(patch_rows=int(want.shape[0]))
