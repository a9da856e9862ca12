"""FPS, radius estimation and patch gathering (a1-a3) on the GPU against float64, on edge inputs and on the route
production runs.

Every entry point is held to the float64 checks of oracle/frontend_cases.py (bounds derived in the docstring of
tests/test_frontend_fp64_cpu.py), evaluated in torch float64 on the device: FPS at every register-tier boundary, in the
throughput forms, several clouds in one launch, device counts over poisoned capacity buffers and the pointnet2 drop-in;
the radius histogram and bisection in the single-cloud and the device-count pair form and on the model's >200000-point
route; patch gathering in the scan, batched, device-count and hash-grid forms (cell coordinates far beyond 4096 per
axis, r = 0) and the ball queries behind the drop-in.  The production route (C2 seed 0, and a C3-sized pair that takes
the hash grid) records every ops.fps / radius_estimate / select_patches_batched call and holds each output to float64.
The largest ratios and the undecided counts are printed with -s and recorded in DESIGN.md section 7."""
import os

import numpy as np
import pytest
import torch

from oracle import frontend_cases as F
from oracle.frontend_cases import merge, report

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


def cu(a, dev, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return t if dtype is None else t.to(dtype)


# ------------------------------------------------------------------------------------------------ a1
TIERS = [4096, 4097, 8192, 8193, 16384, 16385, 24576, 24577, 32768, 32769, 65536, 65537, 131072, 131073, 262144, 262145,
         524288]


def test_fps_tier_boundaries(dev):
    from bufferx_b200 import ops
    acc = {}
    for j, n in enumerate(TIERS):
        xyz = F.fps_cloud("dup" if j % 3 == 1 else "uniform", n, seed=n, offset=1e3 if j % 4 == 3 else 0.0)
        x = cu(xyz, dev)
        idx, kp = ops.fps(x, [0, n], 40)
        merge(acc, F.check_fps(x, 40, idx[0], kp[0]))
    report("fps tier boundaries", acc)


@pytest.mark.parametrize("kind", F.FPS_KINDS)
def test_fps_edge_clouds(dev, kind):
    """npoint 1, N and more than the points left after the skip; N = 1; offsets 1e3 and 1e4 m."""
    from bufferx_b200 import ops
    acc = {}
    for n in (1, 300, 5000):
        for off in ((0.0,) if kind in ("allskip", "fewvalid", "magedge") else (0.0, 1e3, 1e4)):
            x = cu(F.fps_cloud(kind, n, seed=n, offset=off), dev)
            for npoint in sorted({1, n, n + 5, 16} if n <= 300 else {64}):
                idx, kp = ops.fps(x, [0, n], npoint)
                merge(acc, F.check_fps(x, npoint, idx[0], kp[0]))
    report(f"fps {kind}", acc)


def test_fps_throughput_forms_and_mixed_launch(dev):
    """Duplicated-point clouds on the 8-CTA tiers; clouds of mixed sizes and kinds in one launch each pass on their own."""
    from bufferx_b200 import ops
    acc = {}
    for n in (9000, 20000, 40000):
        x = cu(F.fps_cloud("dup", n, seed=n), dev)
        ref, _ = ops.fps(x, [0, n], 96)
        merge(acc, F.check_fps(x, 96, ref[0]))
    clouds = [F.fps_cloud(k, n, seed=i) for i, (k, n) in
              enumerate([("uniform", 1), ("lattice", 700), ("allskip", 50), ("dup", 9000), ("fewvalid", 200), ("uniform", 3000)])]
    off = np.cumsum([0] + [len(c) for c in clouds])
    x = cu(np.concatenate(clouds), dev)
    idx, kp = ops.fps(x, off.tolist(), 64)
    for b, c in enumerate(clouds):
        merge(acc, F.check_fps(x[off[b]:off[b + 1]], 64, idx[b], kp[b]))
    report("fps mixed launch", acc)


def test_fps_device_counts_poisoned_padding(dev):
    """bx_fps_n: capacity buffers whose rows past the count hold NaN; the result must be the exact-size cloud's."""
    from bufferx_b200 import ops
    acc = {}
    caps, counts = [5000, 9000, 300], [4097, 8193, 1]
    clouds = [F.fps_cloud("uniform", c, seed=c) for c in caps]
    for c, n in zip(clouds, counts):
        c[n:] = np.nan
    off = np.cumsum([0] + caps).tolist()
    x = cu(np.concatenate(clouds), dev)
    idx, kp = ops.fps(x, off, 80, d_counts=cu(np.array(counts, np.int32), dev))
    for b, n in enumerate(counts):
        xb = x[off[b]:off[b] + n]
        merge(acc, F.check_fps(xb, 80, idx[b], kp[b]))
        ref, _ = ops.fps(xb.contiguous(), [0, n], 80)
        assert torch.equal(idx[b], ref[0])
    report("fps device counts", acc)


def test_fps_dropin(dev):
    from dropin.pointnet2_ops import pointnet2_utils as pu
    acc = {}
    xyz = np.stack([F.fps_cloud("lattice", 4096, seed=1), F.fps_cloud("uniform", 4096, seed=2, offset=1e4)])
    x = cu(xyz, dev)
    idx = pu.furthest_point_sample(x, 128)
    for b in range(2):
        merge(acc, F.check_fps(x[b], 128, idx[b]))
    report("fps drop-in", acc)


# ------------------------------------------------------------------------------------------------ a2
def _radius_check(dev, kp, pts, ths=F.RADIUS_THRESHOLDS, denom=None):
    from bufferx_b200 import ops
    r, m, hist = ops.radius_estimate(kp, pts, ths, denom=denom)
    lo, hi = F.O.radius_count_bounds(kp, pts)
    denom = denom or pts.shape[0] * kp.shape[0]
    return F.check_radius(hist[:8193].cpu().numpy(), denom, ths, 0.01, m.cpu().numpy(), r.cpu().numpy(), lo, hi)


@pytest.mark.parametrize("kind", F.RADIUS_KINDS)
def test_radius_estimate_vs_fp64(dev, kind):
    kp, pts = F.radius_case(kind, n=20000, kr=500, seed=len(kind))
    out = _radius_check(dev, cu(kp, dev), cu(pts, dev))
    if kind == "axis":
        assert out["hist_undecided_bins"] == 0
    report(f"radius {kind}", out)


@pytest.mark.parametrize("ns,nt", [(9000, 7000), (8000, 8000), (7000, 9000)])
def test_radius_estimate_pair_counts(dev, ns, nt):
    """bx_radius_estimate_n: capacity buffers with NaN past the counts; the source only when ns > nt."""
    from bufferx_b200 import ops
    kps, src = F.radius_case("uniform", n=ns, kr=300, seed=1)
    kpt, tgt = F.radius_case("dense", n=nt, kr=300, seed=2)
    pad = lambda a: np.concatenate([a, np.full((977, 3), np.nan, np.float32)])
    ths = F.RADIUS_THRESHOLDS
    r, m, hist = ops.radius_estimate_pair(cu(kps, dev), cu(pad(src), dev), cu(kpt, dev), cu(pad(tgt), dev), ths,
                                          cu(np.array([ns, nt], np.int32), dev))
    kp, pts = (kps, src) if ns > nt else (kpt, tgt)
    e = F.O.radius_estimation_fp64(cu(src, dev), cu(kps, dev), cu(tgt, dev), cu(kpt, dev), ths)
    out = F.check_radius(hist[:8193].cpu().numpy(), e["denom"], ths, 0.01, m.cpu().numpy(), r.cpu().numpy(), e["lo"], e["hi"])
    r1, m1, _ = ops.radius_estimate(cu(kp, dev), cu(pts, dev), ths)
    assert torch.equal(r, r1) and torch.equal(m, m1)
    report(f"radius pair ns={ns} nt={nt}", out)


def test_radius_subsampled_route_draws_once_per_scale(dev, monkeypatch):
    """BufferX.forward on a pair whose larger cloud has 250000 points: as the reference (BUFFERX.py:320-329, 664-665), each
    scale draws its own 200000 indices from the CPU generator, torch.randint(0, N, (200000,)) in scale order (the same
    indices under torch.manual_seed), builds its histogram on pts[indices] with the denominator keeping N, and takes its
    radius with its own threshold."""
    _subsampled_route(dev, monkeypatch, early_exit=False)


def test_radius_subsampled_route_after_an_early_exit(dev, monkeypatch):
    """The same with early exit on and every pair exiting after scale 0: forward draws the S sub-samples, and leaves
    torch's generator after one draw, where the reference leaves it."""
    _subsampled_route(dev, monkeypatch, early_exit=True)


def _subsampled_route(dev, monkeypatch, early_exit):
    import bufferx_b200 as bx
    from bufferx_b200 import ops
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg("C3")
    cfg.match.enable_early_exit = early_exit
    cfg.match.early_exit_min_inliers = 0          # with early exit on, every pair exits after scale 0
    S, ths_all = cfg.patch.num_scales, list(cfg.patch.search_radius_thresholds)
    model = init_synthetic_weights(bx.BufferX(cfg)).to(dev).eval()
    data = make_pair("C3", 0, n_src=250000, n_tgt=30000)
    draws, calls = [], []
    randint, est = torch.randint, ops.radius_estimate

    def rec_randint(*a, **kw):
        t = randint(*a, **kw)
        draws.append((a, kw, t.clone()))
        return t

    def rec_est(kpts, pts, thresholds, **kw):
        out = est(kpts, pts, thresholds, **kw)
        calls.append((kpts.clone(), pts.clone(), list(thresholds), kw.get("denom"), [o.clone() for o in out]))
        return out

    monkeypatch.setattr(torch, "randint", rec_randint)
    monkeypatch.setattr(ops, "radius_estimate", rec_est)
    torch.manual_seed(1234)
    with torch.no_grad():
        _, _, _, _, _, su = model(data)
    after = torch.get_rng_state()
    monkeypatch.undo()
    assert su == (1 if early_exit else S)
    torch.manual_seed(1234)
    want = [torch.randint(0, 250000, (200000,)) for _ in range(S)]
    sub = [t for a, kw, t in draws if len(a) >= 3 and a[0] == 0 and tuple(a[2]) == (200000,)]
    assert len(sub) == S and all(t.device.type == "cpu" and torch.equal(t, w) for t, w in zip(sub, want)), "not the reference's CPU draws"
    torch.manual_seed(1234)
    for _ in range(su):
        torch.randint(0, 250000, (200000,))
    assert torch.equal(after, torch.get_rng_state()), "the generator is not where the reference leaves it"
    assert len(calls) == S
    src = cu(np.ascontiguousarray(data["src_fds_pcd"], np.float32), dev)
    for i, (kp, pts, ths, denom, (r, m, hist)) in enumerate(calls):
        assert ths == [ths_all[i]], f"scale {i} bisects with {ths}"
        assert denom == 250000 * kp.shape[0] and torch.equal(pts, src[want[i].to(dev)]), f"scale {i} is not on draw {i}"
        lo, hi = F.O.radius_count_bounds(kp, pts)
        report(f"radius model route, 250000 points, scale {i}", F.check_radius(hist[:8193].cpu().numpy(), denom, ths, 0.01,
                                                                             m.cpu().numpy(), r.cpu().numpy(), lo, hi))


def test_radius_subsampled_route_under_capture(dev, monkeypatch):
    """The same pair on a captured slot: the capture must draw the 200000 indices on the device (a host draw would be
    frozen into the graph), and the replay must return a pose."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg("C3")
    model = init_synthetic_weights(bx.BufferX(cfg)).to(dev).eval()
    data = make_pair("C3", 0, n_src=250000, n_tgt=30000)
    draws = []
    randint = torch.randint

    def rec_randint(*a, **kw):
        draws.append((a, kw, torch.cuda.is_current_stream_capturing()))
        return randint(*a, **kw)

    monkeypatch.setattr(torch, "randint", rec_randint)
    with torch.no_grad():
        eager = model(data)
        model.enable_cuda_graphs(True, slots_per_shape=1)
        try:
            out = model.forward_async(data).result()
        finally:
            model.enable_cuda_graphs(False)
    monkeypatch.undo()
    sub = [(kw, cap) for a, kw, cap in draws if len(a) >= 3 and a[0] == 0 and tuple(a[2]) == (200000,)]
    assert sub[0] == ({}, False), "eager forward must draw on the host"
    captured = [kw for kw, cap in sub if cap]
    assert captured and all(torch.device(kw.get("device", "cpu")).type == "cuda" for kw in captured), sub
    for T in (np.asarray(out[0]), np.asarray(eager[0])):
        assert np.isfinite(T).all() and np.abs(T[:3, :3] @ T[:3, :3].T - np.eye(3)).max() < 1e-4


# ------------------------------------------------------------------------------------------------ a3
def _all_forms(dev, pts, kp, r, P, rng, acc, grid_ok=True):
    """Every select_patches entry point on one (cloud, key points, radius): index rows to float64, patches to the mask
    formula, and the batched / device-count / grid forms to the scan form."""
    from bufferx_b200 import ops
    n = len(pts)
    perm = cu(rng.permutation(n).astype(np.int32), dev)
    x, k = cu(pts, dev), cu(kp, dev)
    pts4 = ops.permute_cloud(x, perm)
    pp = pts4[:, :3]
    rd = torch.tensor([r], dtype=torch.float32, device=dev)
    patches, idx = ops.select_patches(pts4, k, r, P, want_idx=True)
    merge(acc, F.check_ball_query(pp, k, r, idx))
    merge(acc, F.check_patches(pp, k, idx, patches))
    p2, i2 = ops.select_patches(pts4, k, rd, P, want_idx=True)
    assert torch.equal(i2, idx) and torch.equal(p2, patches)
    for grid in ((False, True) if grid_ok else (False,)):
        pb = torch.full_like(patches, float("nan"))
        ops.select_patches_batched([(pts4, k, rd)], P, pb, grid=grid)
        merge(acc, F.check_patches(pp, k, idx, pb))
        cap = torch.full((n + 37, 4), float("nan"), device=dev)
        cap[:n] = pts4
        pc = torch.full_like(patches, float("nan"))
        ops.select_patches_batched([(cap, k, rd)], P, pc, grid=grid, d_N=[torch.tensor([n], dtype=torch.int32, device=dev)])
        merge(acc, F.check_patches(pp, k, idx, pc))
    if grid_ok:
        pg, ig = ops.select_patches_grid(pts4, k, rd, P, want_idx=True)
        merge(acc, F.check_ball_query(pp, k, r, ig))
        merge(acc, F.check_patches(pp, k, ig, pg))
        assert torch.equal(ig, idx) and torch.equal(pg, patches), "hash grid != scan"
    return idx


# (radius, power-of-two cell value the cloud straddles): the window of 3 cells (2^13), of up to 4 (2^16 .. 2^20), and the
# whole-cloud scan beyond 2^21 cells (2^22)
STRADDLE = [(0.09, 13), (0.77, 16), (0.09, 17), (0.05, 18), (0.3, 19), (0.05, 20), (0.05, 22)]


@pytest.mark.parametrize("radius,k", STRADDLE)
def test_select_patches_grid_across_power_of_two_cells(dev, radius, k):
    """Clouds whose cell values (v / (1.001 r)) straddle 2^k on every axis, on both sides of the origin: fp32 rounding of
    the cell value puts hits two cells from their key point there.  Planted: the pairs (cells 131071 / 131073 at
    r = 0.09, 262143 / 262145 at r = 0.05) that the +-1 cell query missed.  Every form equal to the scan and float64."""
    acc = {}
    rng = np.random.default_rng(k)
    cell = float(np.float32(np.float32(radius) * np.float32(1.001)))
    for sgn in (1.0, -1.0):
        c = sgn * 2.0 ** k * cell
        kp = (c + rng.uniform(-3 * radius, 3 * radius, (96, 3))).astype(np.float32)
        v = rng.normal(size=(3000, 3))
        v /= np.linalg.norm(v, axis=1, keepdims=True)
        v[:1500] = np.eye(3)[rng.integers(0, 3, 1500)] * rng.choice([-1.0, 1.0], (1500, 1))
        pts = (kp[rng.integers(0, 96, 3000)].astype(np.float64) + v * rng.uniform(0.9, 1.0, (3000, 1)) * radius).astype(np.float32)
        for r0, qx, px in ((0.09, 11808.27734375, 11808.3671875), (0.05, 13120.3076171875, 13120.357421875)):
            if r0 == radius and (sgn * qx) / cell > 0 and abs(abs(qx / cell) - 2.0 ** k) < 4:
                kp[0] = (sgn * qx, kp[0, 1], kp[0, 2])
                pts[0] = (sgn * px, kp[0, 1], kp[0, 2])
                acc["planted"] = acc.get("planted", 0) + 1
        _all_forms(dev, pts, kp, radius, 64, rng, acc)
    if (radius, k) in ((0.09, 17), (0.05, 18)):
        assert acc.get("planted") == 1
    report(f"patches across 2^{k} cells, r = {radius}", acc)


@pytest.mark.parametrize("kind", F.PATCH_KINDS)
@pytest.mark.parametrize("offset,r", [(0.0, None), (1e3, 0.1), (1e4, 0.05)])
def test_select_patches_vs_fp64(dev, kind, offset, r):
    """Offsets up to 1e4 m with r down to 0.05: 2e5 cells per axis in the hash grid, beyond the 4096 the CPU probe
    covers; r = 0 (inf cells) on every case."""
    acc = {}
    rng = np.random.default_rng(2)
    P = 32
    pts, kp, rr = F.patch_case(kind, n=5000, k=96, r=r or 0.3, P=P, seed=4, offset=offset)
    for radius in (rr, 0.0):
        _all_forms(dev, pts, kp, radius, P, rng, acc)
    report(f"patches {kind} offset {offset:g}", acc)


def test_select_patches_grid_threshold_sizes(dev):
    """N at GRID_MIN_POINTS - 1, GRID_MIN_POINTS and + 1 (the model switches between scan and grid there)."""
    from bufferx_b200 import ops
    acc = {}
    rng = np.random.default_rng(3)
    g = ops.GRID_MIN_POINTS
    for n in (g - 1, g, g + 1):
        pts, kp, r = F.patch_case("uniform", n=n, k=200, r=0.12, seed=n)
        _all_forms(dev, pts, kp, r, 64, rng, acc)
    report("patches around GRID_MIN_POINTS", acc)


def test_ball_query_entry_points(dev):
    """bx_ball_query and bx_ball_query_batched at N = 4096 (shared-memory path) and 4097 (global path), and through
    the drop-in's ball_query."""
    from bufferx_b200 import ops
    from dropin.pointnet2_ops import pointnet2_utils as pu
    acc = {}
    for n in (4096, 4097):
        for kind in ("exact", "counts", "cells"):
            pts, kp, r = F.patch_case(kind, n=n, k=64, r=0.2, P=16, seed=n)
            pts = pts[:n]
            x, q = cu(pts, dev), cu(kp, dev)
            idx = ops.ball_query(x, q, r, 16)
            merge(acc, F.check_ball_query(x, q, r, idx))
            xb = torch.stack([x, x.flip(0)])
            qb = torch.stack([q, q])
            ib = ops.ball_query_batched(xb, qb, r, 16)
            assert torch.equal(ib[0], idx)
            merge(acc, F.check_ball_query(xb[1], q, r, ib[1]))
            assert torch.equal(pu.ball_query(r, 16, xb, qb).to(torch.int32), ib)
    report("ball query entry points", acc)


# ------------------------------------------------------------------------------------------------ production route
def _route(dev, oracle, monkeypatch, name, n_src=None, n_tgt=None, pair_seed=0, key_stride=1):
    import bufferx_b200 as bx
    from bufferx_b200 import ops
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg(name)
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=(name == "C2")).to(dev).eval()
    data = make_pair(name, pair_seed, n_src=n_src, n_tgt=n_tgt)
    perms = oracle.draw_perms(cfg, data["src_fds_pcd"].shape[0], data["tgt_fds_pcd"].shape[0], pair_seed)
    rec = {"fps": [], "radius_estimate": [], "radius_estimate_pair": [], "select_patches_batched": []}
    orig = {k: getattr(ops, k) for k in rec}

    def clone(x):
        if isinstance(x, torch.Tensor):
            return x.clone()
        if isinstance(x, (list, tuple)):
            return type(x)(clone(y) for y in x)
        return x

    def wrap(name_):
        def f(*a, **kw):
            inp = clone(list(a))
            r = orig[name_](*a, **kw)
            outs = r if isinstance(r, tuple) else (r,)
            rec[name_].append((inp, dict(kw), clone(list(outs))))     # select_patches_batched: outs = [the filled patches]
            return r
        return f

    for k in rec:
        monkeypatch.setattr(ops, k, wrap(k))
    with torch.no_grad():
        model(data, perms=perms, ransac_seed=0)
    torch.cuda.synchronize()
    for k in rec:
        monkeypatch.setattr(ops, k, orig[k])
    acc = {}
    # FPS: one launch for both clouds
    assert len(rec["fps"]) == 1, len(rec["fps"])
    (xyz, offs, npoint), _, (idx, kp) = rec["fps"][0][0][:3], rec["fps"][0][1], rec["fps"][0][2]
    assert len(offs) == 3
    for b in range(2):
        merge(acc, F.check_fps(xyz[offs[b]:offs[b + 1]], npoint, idx[b], kp[b]))
    # radius: the eager route, one histogram
    assert len(rec["radius_estimate"]) == 1 and not rec["radius_estimate_pair"]
    (kpr, ptr, ths), kw, (r, m, hist) = rec["radius_estimate"][0][0][:3], rec["radius_estimate"][0][1], rec["radius_estimate"][0][2]
    lo, hi = F.O.radius_count_bounds(kpr, ptr)
    merge(acc, F.check_radius(hist[:8193].cpu().numpy(), kw["denom"], ths, 0.01, m.cpu().numpy(), r.cpu().numpy(), lo, hi))
    # patches: every job of every call, scan or grid by the cloud size
    assert rec["select_patches_batched"]
    for (jobs, P, _), kw, (patches,) in rec["select_patches_batched"]:
        assert kw.get("d_K") is None and kw.get("d_N") is None
        want_grid = all(j[0].shape[0] >= ops.GRID_MIN_POINTS for j in jobs)
        assert kw.get("grid", False) == want_grid
        acc["grid_calls"] = acc.get("grid_calls", 0) + int(want_grid)
        o = 0
        for pts4, kpts, rd in jobs:
            K = kpts.shape[0]
            sel = slice(0, K, key_stride)
            _, idx_s = orig_select(pts4, kpts[sel].contiguous(), rd, P)
            merge(acc, F.check_ball_query(pts4[:, :3], kpts[sel], float(rd.item()), idx_s))
            merge(acc, F.check_patches(pts4[:, :3], kpts[sel], idx_s, patches[o:o + K][sel]))
            o += K
    return acc, data, rec


def orig_select(pts4, kpts, rd, P):
    from bufferx_b200 import ops
    return ops.select_patches(pts4, kpts, rd, P, want_idx=True)


def test_production_route_c2(dev, oracle, monkeypatch):
    """BufferX.forward on the C2 seed-0 pair (20000 points per cloud: all six jobs through the hash grid in one
    batched call): the FPS, radius and patch calls to float64; the golden des_r / s_fps / t_fps of c2_seed0.npz to
    float64 as well."""
    acc, data, rec = _route(dev, oracle, monkeypatch, "C2")
    assert len(rec["select_patches_batched"]) == 1 and acc["grid_calls"] == 1
    g = np.load(f"{ROOT}/tests/golden/c2_seed0.npz")
    (xyz, offs, npoint), _, (idx, kp) = rec["fps"][0][0][:3], rec["fps"][0][1], rec["fps"][0][2]
    for b, key in enumerate(("s_fps", "t_fps")):
        gi = g[key].reshape(-1)
        merge(acc, F.check_fps(xyz[offs[b]:offs[b + 1]], len(gi), gi))
    (kpr, ptr, ths), kw, (r, m, hist) = rec["radius_estimate"][0][0][:3], rec["radius_estimate"][0][1], rec["radius_estimate"][0][2]
    lo, hi = F.O.radius_count_bounds(kpr, ptr)
    for i, th in enumerate(ths):
        reach, und, radii = F.O.radius_fp64(lo, hi, kw["denom"], th, 0.01)
        assert np.float32(g["des_r"].reshape(-1)[i]) in set(radii.values())
    report("production route C2 seed 0", acc)


def test_production_route_c3_sized_grid(dev, oracle, monkeypatch):
    """A C3-sized pair (120000 / 100000 points): the hash-grid route; every eighth key point's row to float64."""
    acc, _, rec = _route(dev, oracle, monkeypatch, "C3", n_src=120000, n_tgt=100000, key_stride=8)
    assert len(rec["select_patches_batched"]) == 1 and acc["grid_calls"] == 1
    report("production route C3-sized", acc)
