"""GPU parity: every CUDA stage against the CPU oracle on identical inputs, through the C-ABI
(``bufferx_b200.ops`` -> ctypes -> libbufferx_b200.so).  Integer / index results must be bit-exact;
floating point within the tolerance written next to each assert (descriptors 1e-4 rel, north_star)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


def cu(a, dev, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.to(dtype)
    return t.to(dev).contiguous()


def relerr(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


# ------------------------------------------------------------------------------------------------ a1
@pytest.mark.parametrize("n,m,kind", [(300, 64, "dup"), (5000, 2000, "plain"), (20000, 2000, "plain"),
                                      (20000, 300, "dup"), (40000, 200, "plain"), (70000, 128, "plain"),
                                      (120000, 96, "plain"), (200000, 24, "plain"), (300000, 12, "dup")])
def test_fps_bit_exact(dev, oracle, n, m, kind):
    from bufferx_b200 import ops
    rng = np.random.default_rng(n + m)
    xyz = rng.uniform(-3, 3, size=(n, 3)).astype(np.float32)
    if kind == "dup":                       # exact ties + candidates the |p|^2 <= 1e-3 rule must skip
        xyz[n // 2:] = xyz[: n - n // 2]
        xyz[5] = [0.01, 0.02, 0.01]
        xyz[n - 1] = [0.0, 0.0, 0.0]
    idx, kp = ops.fps(cu(xyz, dev), [0, n], m)
    exp = oracle.fps(xyz, m)
    got = idx[0].cpu().numpy()
    assert (got == exp).all(), f"first mismatch at {np.flatnonzero(got != exp)[:5]}"
    assert (kp[0].cpu().numpy() == xyz[exp]).all()


@pytest.mark.parametrize("n,m", [(20000, 1500), (120000, 300), (5000, 512)])
def test_fps_mbarrier_exchange_equals_cluster_sync_exchange(dev, oracle, n, m):
    """The production cluster exchange (remote st.shared::cluster + mbarrier.arrive.release.cluster, local acquire wait) and
    the verification form (the same stores ordered by cluster.sync(), which racecheck models)
    give the same indices -- and both equal the oracle."""
    from bufferx_b200 import ops
    lib = ops.load_library()
    rng = np.random.default_rng(n)
    xyz = rng.normal(size=(n, 3)).astype(np.float32)
    d = cu(xyz, dev)
    old = lib.bx_fps_set_sync_mode(1)
    try:
        a, _ = ops.fps(d, [0, n], m)                 # cluster.sync() exchange (racecheck-clean reference form)
        lib.bx_fps_set_sync_mode(0)
        b, _ = ops.fps(d, [0, n], m)                 # st.async + transaction-count mbarrier (production)
        lib.bx_fps_set_sync_mode(2)
        c, _ = ops.fps(d, [0, n], m)                 # remote stores + mbarrier arrive / acquire wait (round 1)
    finally:
        lib.bx_fps_set_sync_mode(old)
    assert torch.equal(a, b) and torch.equal(a, c) and (a[0].cpu().numpy() == oracle.fps(xyz, m)).all()


@pytest.mark.parametrize("n,m", [(20000, 700), (7000, 300), (40000, 200), (4097, 64)])
@pytest.mark.parametrize("cl", [2, 4])
def test_fps_throughput_form_same_indices(dev, oracle, n, m, cl):
    """bx_fps_ex with 2 / 4 CTAs per cloud (the form BufferX uses with several pairs in flight): the indices of the default
    8-CTA form and of the oracle, incl. exact ties (duplicated points)."""
    from bufferx_b200 import ops
    rng = np.random.default_rng(n + cl)
    xyz = rng.normal(size=(n, 3)).astype(np.float32)
    xyz[n // 2:n // 2 + 50] = xyz[:50]                                   # exact duplicates: tie-breaking by rank
    d = cu(np.concatenate([xyz, xyz[::-1]]), dev)                        # two clouds in one launch
    a, ka = ops.fps(d, [0, n, 2 * n], m)
    b, kb = ops.fps(d, [0, n, 2 * n], m, max_cluster=cl)
    assert torch.equal(a, b) and torch.equal(ka, kb)
    assert (b[0].cpu().numpy() == oracle.fps(xyz, m)).all()


def test_fps_two_clouds_one_launch(dev, oracle):
    from bufferx_b200 import ops
    rng = np.random.default_rng(0)
    a = rng.normal(size=(7000, 3)).astype(np.float32)
    b = rng.normal(size=(3000, 3)).astype(np.float32) * 2
    idx, _ = ops.fps(cu(np.concatenate([a, b]), dev), [0, 7000, 10000], 500)
    assert (idx[0].cpu().numpy() == oracle.fps(a, 500)).all() and (idx[1].cpu().numpy() == oracle.fps(b, 500)).all()


# ------------------------------------------------------------------------------------------------ a2
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_radius_estimate_matches_oracle(dev, oracle, seed):
    from bufferx_b200 import ops
    rng = np.random.default_rng(seed)
    n = [6000, 20000, 9000][seed]
    pts = (rng.uniform(-3, 3, size=(n, 3)) * [1, 1, 0.4]).astype(np.float32)
    kp = pts[oracle.fps(pts, 500)]
    r, m, hist = ops.radius_estimate(cu(kp, dev), cu(pts, dev), [5, 2, 0.5])
    cum = oracle.radius_hist(kp, pts)
    assert (hist[:8193].cpu().numpy().astype(np.int64) == cum).all()      # cumulative histogram is bit-exact
    exp = oracle.radius_estimation(pts[:1], kp[:1], pts, kp, [5, 2, 0.5], cum=cum)
    assert np.allclose(r.cpu().numpy(), np.array(exp, dtype=np.float32), atol=0)


# ------------------------------------------------------------------------------------------------ a3
@pytest.mark.parametrize("radius,P", [(0.35, 64), (1.2, 512), (0.02, 32), (50.0, 128)])
def test_select_patches_bit_exact(dev, oracle, radius, P):
    from bufferx_b200 import ops
    rng = np.random.default_rng(int(radius * 100) + P)
    n, K = 9000, 300
    pts = (rng.uniform(-3, 3, size=(n, 3)) * [1, 1, 0.3]).astype(np.float32)
    perm = rng.permutation(n).astype(np.int32)
    kp = pts[oracle.fps(pts, K)]
    pts4 = ops.permute_cloud(cu(pts, dev), cu(perm, dev))
    assert (pts4[:, :3].cpu().numpy() == pts[perm]).all()
    eidx, epat = oracle.select_patches(pts, perm, kp, radius, P)
    pat, idx = ops.select_patches(pts4, cu(kp, dev), radius, P, want_idx=True)
    assert (idx.cpu().numpy() == eidx).all()
    assert (pat.cpu().numpy() == epat).all()
    # device-side radius gives the same result
    pat2, _ = ops.select_patches(pts4, cu(kp, dev), torch.tensor([radius], dtype=torch.float32, device=dev), P)
    assert (pat2.cpu().numpy() == epat).all()


@pytest.mark.parametrize("n,K,radius,P", [(60000, 300, 0.35, 512), (60000, 64, 0.02, 64), (131073, 100, 0.6, 512), (9000, 50, 5.0, 128)])
def test_select_patches_grid_equals_scan(dev, oracle, n, K, radius, P):
    """bx_select_patches_grid (spatial hash + per-key-point index bitmap) against the streaming scan and, at the small size,
    the oracle: identical index rows and patches -- dense balls (more than P hits), empty balls, a radius larger than the cloud
    (every bucket aliased), N not a multiple of 32, negative coordinates."""
    from bufferx_b200 import ops
    rng = np.random.default_rng(n + K)
    pts = (rng.uniform(-3, 3, size=(n, 3)) * [1, 1, 0.3]).astype(np.float32)
    perm = rng.permutation(n).astype(np.int32)
    kp = pts[rng.choice(n, K, replace=False)]
    kp[0] = [40.0, 40.0, 40.0]                                           # a key-point far outside the cloud: no hit at all
    pts4 = ops.permute_cloud(cu(pts, dev), cu(perm, dev))
    rad = torch.tensor([radius], dtype=torch.float32, device=dev)
    pa, ia = ops.select_patches(pts4, cu(kp, dev), rad, P, want_idx=True)
    pb, ib = ops.select_patches_grid(pts4, cu(kp, dev), rad, P, want_idx=True)
    assert torch.equal(ia, ib) and torch.equal(pa, pb)
    if n <= 10000:
        eidx, epat = oracle.select_patches(pts, perm, kp, radius, P)
        assert (ib.cpu().numpy() == eidx).all() and (pb.cpu().numpy() == epat).all()


def test_select_patches_batched_equals_per_job(dev, oracle):
    """bx_select_patches_batched (all (cloud, scale) jobs of a pair in one launch) against the oracle job by job: different
    clouds, key-point counts (one not a multiple of the 4 key-points of a CTA) and radii, incl. an empty-ball radius."""
    from bufferx_b200 import ops
    rng = np.random.default_rng(77)
    P, jobs, expect = 128, [], []
    for n, K, radius in ((9000, 300, 0.5), (5000, 157, 0.9), (9000, 300, 0.01), (2049, 1, 3.0)):
        pts = (rng.uniform(-3, 3, size=(n, 3)) * [1, 1, 0.3]).astype(np.float32)
        perm = rng.permutation(n).astype(np.int32)
        kp = pts[oracle.fps(pts, K)]
        jobs.append((ops.permute_cloud(cu(pts, dev), cu(perm, dev)), cu(kp, dev), torch.tensor([radius], dtype=torch.float32, device=dev)))
        expect.append(oracle.select_patches(pts, perm, kp, radius, P)[1])
    for grid in (False, True):          # streaming scan / hash grid, all jobs in one launch (per phase)
        out = torch.full((sum(j[1].shape[0] for j in jobs), P, 3), float("nan"), dtype=torch.float32, device=dev)
        ops.select_patches_batched(jobs, P, out, grid=grid)
        assert (out.cpu().numpy() == np.concatenate(expect)).all(), f"grid={grid}"


def test_ball_query_bit_exact(dev, oracle):
    from bufferx_b200 import ops
    rng = np.random.default_rng(9)
    xyz = rng.uniform(-1, 1, size=(777, 3)).astype(np.float32)
    q = np.concatenate([xyz[:40], [[9, 9, 9]]]).astype(np.float32)
    idx = ops.ball_query(cu(xyz, dev), cu(q, dev), 0.3, 10)
    assert (idx.cpu().numpy() == oracle.ball_query(xyz, q, 0.3, 10)[0]).all()


# ------------------------------------------------------------------------------------------- a4+a5
@pytest.mark.parametrize("aligned", [False, True])
def test_lrf_bit_exact(dev, oracle, c1, aligned):
    from bufferx_b200 import ops
    patches = c1["res"][5]["scales"][0]["src"]["patches"]
    des_r = c1["res"][5]["des_r"][0]
    delta, Rt, ra = ops.lrf(cu(patches, dev), des_r, aligned)
    ed, eR, era = oracle.lrf(patches, des_r, aligned)
    assert (Rt.cpu().numpy() == eR).all(), f"R max diff {np.abs(Rt.cpu().numpy() - eR).max()}"
    assert (ra.cpu().numpy() == era).all()
    assert (delta.cpu().numpy() == ed).all()
    if not aligned:       # sanity: R is a rotation taking the z-axis onto +z
        R = Rt.cpu().numpy().astype(np.float64)
        assert np.abs(R @ R.transpose(0, 2, 1) - np.eye(3)).max() < 1e-5


# ------------------------------------------------------------------------------------------- a6+a7
def test_spt_pnt(dev, oracle, c1):
    import bufferx_b200 as bx
    from bufferx_b200 import ops
    aux = c1["res"][5]
    delta = aux["scales"][0]["src"]["delta"]
    model = c1["model"].to(dev)
    prep = model.Desc.prepared(dev)
    assert (prep["voxels"].cpu().numpy() == oracle.voxel_table()).all()
    assert (prep["rot"].cpu().numpy() == oracle.derot_table()).all()
    feat, vidx, inv = ops.spt_pnt(cu(delta, dev), prep["voxels"], prep["rot"], 0.8 / 3, 10, prep["w_pnt"], prep["b_pnt"], 20, debug=True)
    einv, evidx = oracle.spt(delta)
    assert (vidx.cpu().numpy() == evidx).all()                       # integer selection: bit-exact
    assert (inv.cpu().numpy() == einv).all()                         # de-rotated samples: bit-exact
    with torch.no_grad():
        efeat = oracle.pnt_max(torch.from_numpy(einv), c1["sd"]).numpy()
    assert feat.shape == (delta.shape[0], 4, 420, 4)                 # channel-blocked, the layout bx_conv_layer_tc reads
    feat = ops.from_blocked(feat)
    assert np.abs(feat.cpu().numpy() - efeat).max() < 2e-6 * max(1.0, np.abs(efeat).max())   # folded BN: fp32 rounding only
    model.cpu()


# ------------------------------------------------------------------------------------------- a8+a9
def test_spt_presplit_output_is_the_split_of_the_fp32_features(dev, oracle, c1):
    """bx_spt_pnt_sd writes the features directly in the presplit padded fp16 format of the conv kernel: bit-identical to
    splitting bx_spt_pnt's fp32 features (hi = fp16(x), lo = fp16((x - hi) * 2^11)), zero rows and wrap columns included."""
    from bufferx_b200 import ops
    delta = c1["res"][5]["scales"][0]["src"]["delta"]
    K = delta.shape[0]
    prep = c1["model"].to(dev).Desc.prepared(dev)
    d = cu(delta, dev)
    feat = ops.spt_pnt(d, prep["voxels"], prep["rot"], 0.8 / 3, 10, prep["w_pnt"], prep["b_pnt"], 20)
    img = ops.spt_pnt_sd(d, prep["voxels"], prep["rot"], 0.8 / 3, 10, prep["w_pnt"], prep["b_pnt"], 20)
    x = ops.from_blocked(feat).view(K, 16, 3, 140).permute(0, 2, 1, 3).reshape(K, 48, 7, 20)      # chunk = radial slice
    want = ops.sd_pack(x)
    rows = K * 176 + 22
    assert img.shape == want.shape and torch.equal(img[:, :, :rows].view(torch.int16), want[:, :, :rows].view(torch.int16))
    c1["model"].cpu()


def test_cylindrical_net_and_both_pooling_layouts(dev, oracle, c1):
    """The descriptor stack (channel-blocked fp32 in / out) against the oracle, and the pooling kernel from the channel-first
    and the channel-blocked input layout: both against the oracle, and bit-identical to each other."""
    from bufferx_b200 import ops
    aux = c1["res"][5]
    s = aux["scales"][0]["src"]
    model = c1["model"].to(dev)
    K = s["feat"].shape[0]
    f = cu(s["feat"].numpy(), dev)                                   # oracle layout: [K,16,420]
    ex = s["x"].numpy()
    prep = model.Desc.prepared(dev)
    x, _ = model.Desc.conv_net(ops.to_blocked(f))                    # channel-blocked in / out: [K,8,140,4]
    assert x.shape == (K, 8, 140, 4)
    xcf = ops.from_blocked(x).reshape(K, 32, 7, 20)
    d2, e2 = ops.pool_desc(ops.to_blocked(cu(ex, dev).reshape(K, 32, 140)), prep["w1"], prep["b1"], prep["w2"], prep["b2"],
                           channels_last=True)
    assert relerr(xcf.cpu().numpy(), ex) < 1e-4                      # 8 stacked fp32 convs vs torch CPU
    desc, equi = ops.pool_desc(cu(ex, dev), prep["w1"], prep["b1"], prep["w2"], prep["b2"])
    assert np.abs(desc.cpu().numpy() - s["desc"].numpy()).max() < 1e-5
    assert np.abs(equi.cpu().numpy() - s["equi"].numpy()).max() < 1e-5
    assert (d2 == desc).all() and (e2 == equi).all()                 # both input layouts of the pooling kernel agree bit for bit
    model.cpu()


# ---------------------------------------------------------------------------------------------- a10
@pytest.mark.parametrize("Ka,Kb", [(256, 256), (1500, 1500), (70, 901)])
def test_mutual_nn_bit_exact(dev, oracle, Ka, Kb):
    from bufferx_b200 import ops
    rng = np.random.default_rng(Ka + Kb)
    a = rng.normal(size=(Ka, 32)).astype(np.float32)
    b = rng.normal(size=(Kb, 32)).astype(np.float32)
    a /= np.linalg.norm(a, axis=1, keepdims=True)
    b /= np.linalg.norm(b, axis=1, keepdims=True)
    b[Kb // 2] = b[3]                                                # exact tie
    a[5] = b[7]
    s, t, dM, snn, tnn = ops.mutual_nn(cu(a, dev), cu(b, dev), want_nn=True)
    es, et, esnn, etnn = oracle.mutual_nn(a, b)
    M = int(dM.item())
    assert (snn.cpu().numpy()[:Ka] == esnn).all() and (tnn.cpu().numpy()[:Kb] == etnn).all()
    assert M == len(es) and (s[:M].cpu().numpy() == es).all() and (t[:M].cpu().numpy() == et).all()


# ------------------------------------------------------------------------------------------ a11-a12
def test_cost_volume_and_hypotheses(dev, oracle, c1):
    from bufferx_b200 import ops
    aux = c1["res"][5]
    sc = aux["scales"][0]
    model = c1["model"].to(dev)
    K = sc["src"]["desc"].shape[0]
    es, et = cu(sc["src"]["equi"].numpy(), dev), cu(sc["tgt"]["equi"].numpy(), dev)
    sm, tm = cu(sc["s_mids"], dev, torch.int32), cu(sc["t_mids"], dev, torch.int32)
    M = len(sc["s_mids"])
    smp = torch.zeros(K, dtype=torch.int32, device=dev); smp[:M] = sm
    tmp = torch.zeros(K, dtype=torch.int32, device=dev); tmp[:M] = tm
    dM = torch.tensor([M], dtype=torch.int32, device=dev)
    logits = model.Pose.logits(es, et, smp, tmp, dM, K)
    cfg = c1["cfg"]
    src_k = c1["data"]["src_fds_pcd"][aux["s_fps"][:K]]
    tgt_k = c1["data"]["tgt_fds_pcd"][aux["t_fps"][:K]]
    offs = torch.zeros(2, dtype=torch.int32, device=dev)
    ind = torch.zeros(K, dtype=torch.float32, device=dev)
    Ra, ta = torch.zeros((K, 3, 3), device=dev), torch.zeros((K, 3), device=dev)
    ssa, tta = torch.zeros((K, 3), device=dev), torch.zeros((K, 3), device=dev)
    ops.hypotheses(logits, 20, cu(src_k, dev), cu(tgt_k, dev), cu(sc["src"]["R"].numpy(), dev), cu(sc["tgt"]["R"].numpy(), dev),
                   smp, tmp, dM, K, offs[0:1], offs[1:2], ind, Ra, ta, ssa, tta)
    assert int(offs[1].item()) == M
    assert np.abs(ind[:M].cpu().numpy() - sc["ind"]).max() < 2e-3     # soft arg-max bin (0..19) after 10 fp32 convs
    # hypotheses from the ORACLE's bins must agree tightly: recompute with oracle ind through torch
    R, t = oracle.hypotheses(ind[:M].cpu(), torch.from_numpy(src_k)[sc["s_mids"].astype(np.int64)],
                             torch.from_numpy(tgt_k)[sc["t_mids"].astype(np.int64)], sc["src"]["R"][sc["s_mids"].astype(np.int64)],
                             sc["tgt"]["R"][sc["t_mids"].astype(np.int64)], 20)
    assert np.abs(Ra[:M].cpu().numpy() - R.numpy()).max() < 5e-6 and np.abs(ta[:M].cpu().numpy() - t.numpy()).max() < 5e-5
    assert (ssa[:M].cpu().numpy() == src_k[sc["s_mids"]]).all() and (tta[:M].cpu().numpy() == tgt_k[sc["t_mids"]]).all()
    model.cpu()


# ---------------------------------------------------------------------------------------------- a13
def _corr_problem(rng, n, inlier_frac, noise=0.01):
    ss = rng.uniform(-3, 3, (n, 3))
    A = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    A *= np.sign(np.linalg.det(A))
    tv = rng.uniform(-1, 1, 3)
    tt = ss @ A.T + tv + rng.normal(scale=noise, size=(n, 3))
    out = rng.random(n) > inlier_frac
    tt[out] = rng.uniform(-3, 3, (out.sum(), 3))
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = A, tv
    return ss.astype(np.float32), tt.astype(np.float32), T, ~out


@pytest.mark.parametrize("Mc", [1, 37, 1200, 4500])
def test_consensus_bit_exact(dev, oracle, Mc):
    from bufferx_b200 import ops
    rng = np.random.default_rng(Mc)
    ss, tt, T, inl = _corr_problem(rng, Mc, 0.4, 0.02)
    R = np.tile(np.eye(3, dtype=np.float32), (Mc, 1, 1))
    t = rng.normal(size=(Mc, 3)).astype(np.float32)
    for j in range(0, Mc, 3):           # a third of the hypotheses are the true pose + small perturbation
        R[j] = T[:3, :3].astype(np.float32)
        t[j] = (T[:3, 3] + rng.normal(scale=0.02, size=3)).astype(np.float32)
    cap = Mc + 11
    pad = lambda a: np.concatenate([a, np.zeros((cap - Mc,) + a.shape[1:], a.dtype)])
    ind, dI, dbest, counts = ops.consensus(cu(pad(ss), dev), cu(pad(tt), dev), cu(pad(R), dev), cu(pad(t), dev),
                                           torch.tensor([Mc], dtype=torch.int32, device=dev), cap, 20, 1 / 3)
    eind, ebest, ecounts = oracle.consensus(ss, tt, R, t, 20, 1 / 3)
    assert (counts[:Mc].cpu().numpy() == ecounts).all()
    assert int(dbest.item()) == ebest and int(dI.item()) == len(eind)
    assert (ind[:len(eind)].cpu().numpy() == eind).all()


# ---------------------------------------------------------------------------------------------- a14
@pytest.mark.parametrize("n,frac,conf,iters", [(400, 0.5, 0.999, 50000), (300, 0.15, 1.0, 20000), (60, 0.3, 0.999, 50000),
                                               (1000, 0.05, 0.999, 50000), (2, 1.0, 0.999, 100), (0, 1.0, 0.999, 100)])
def test_ransac_equals_oracle(dev, oracle, n, frac, conf, iters):
    from bufferx_b200 import ops
    rng = np.random.default_rng(n + iters)
    total = max(n, 3) + 40
    ss, tt, T, _ = _corr_problem(rng, total, frac)
    ind = np.sort(rng.choice(total, n, replace=False)).astype(np.int32) if n else np.zeros(0, np.int32)
    pad = np.zeros(max(n, 1) + 5, np.int32)
    pad[:n] = ind
    res = ops.ransac(cu(ss, dev), cu(tt, dev), cu(pad, dev), torch.tensor([n], dtype=torch.int32, device=dev), len(pad),
                     0.10, 0.8, conf, iters, seed=1234)
    Tg, ninl, bitr, nit = ops.decode_ransac_result(res.cpu())
    e = oracle.ransac(ss, tt, ind, 0.10, 0.8, conf, iters, 1234)
    assert ninl == e["num_inliers"] and bitr == e["best_itr"] and nit == e["iters"], (ninl, bitr, nit, e["num_inliers"], e["best_itr"], e["iters"])
    assert np.abs(Tg - e["T"]).max() < 1e-12


def test_ransac_statistical_success(dev):
    """Open3D-equivalent acceptance on many seeds: the recovered pose is inside the RRE/RTE thresholds."""
    from bufferx_b200 import ops
    from bufferx_b200.se3 import compute_rre, compute_rte
    rng = np.random.default_rng(5)
    ss, tt, T, inl = _corr_problem(rng, 500, 0.3)
    d_ss, d_tt = cu(ss, dev), cu(tt, dev)
    ind = torch.arange(500, dtype=torch.int32, device=dev)
    dI = torch.tensor([500], dtype=torch.int32, device=dev)
    ok = 0
    for seed in range(20):
        Tg, ninl, _, _ = ops.decode_ransac_result(ops.ransac(d_ss, d_tt, ind, dI, 500, 0.10, 0.8, 0.999, 50000, seed).cpu())
        ok += compute_rre(Tg, T) < 15.0 and compute_rte(Tg, T) < 0.3 and ninl > 0.7 * inl.sum()
    assert ok == 20


# ---------------------------------------------------------------------------------------------- a15
def test_refine_close_to_oracle(dev, oracle):
    from bufferx_b200 import ops
    rng = np.random.default_rng(8)
    ss, tt, T, _ = _corr_problem(rng, 900, 0.6)
    T0 = T.copy()
    T0[:3, 3] += 0.03
    To, rounds = ops.refine(cu(ss, dev), cu(tt, dev), torch.tensor([900], dtype=torch.int32, device=dev), 900,
                            cu(T0.reshape(16), dev, torch.float64), 0.10)
    eT, erounds = oracle.refine(ss, tt, T0.astype(np.float32), 0.10)
    assert np.abs(To.cpu().numpy().reshape(4, 4) - eT).max() < 1e-5      # fp32 pose, fp64 fit: summation order only
    assert int(rounds.item()) == erounds


# ------------------------------------------------------------------------------------------- whole pair
def _rel_rows(a, b):
    den = np.abs(b).max(1)
    return np.abs(a - b).max(1) / np.where(den > 0, den, 1)


def _compare_pair(model, sd, cfg, data, perms, oracle, name):
    from bufferx_b200.se3 import compute_rre, compute_rte
    with torch.no_grad():
        pose, times, ninl, nmut, nind, su = model(data, perms=perms, ransac_seed=0, debug=True)
    dbg = model.last_debug
    o_pose, o_ninl, o_nmut, o_nind, o_su, aux = oracle.register_pair(sd, cfg, data, perms, 0, keep=True)
    K = cfg.patch.num_fps
    assert (dbg["fps_idx"][0].cpu().numpy()[:len(aux["s_fps"])] == aux["s_fps"]).all()
    assert (dbg["fps_idx"][1].cpu().numpy()[:len(aux["t_fps"])] == aux["t_fps"]).all()
    assert np.allclose(dbg["des_r"].cpu().numpy(), np.array(aux["des_r"], dtype=np.float32), atol=0)
    rep = {}
    worst = 0.0
    for i, (sc, osc) in enumerate(zip(dbg["scales"], aux["scales"])):
        for side, key in (("s", "src"), ("t", "tgt")):
            assert (sc[side]["idx"].cpu().numpy() == osc[key]["idx"]).all(), f"{name} scale {i} {key}: neighbour lists differ"
            assert (sc[side]["vidx"].cpu().numpy() == osc[key]["vidx"]).all(), f"{name} scale {i} {key}: voxel selections differ"
            assert (sc[side]["R"].cpu().numpy() == osc[key]["R"].numpy()).all()
            d, od = sc[side]["desc"].cpu().numpy(), osc[key]["desc"].numpy()
            rel = _rel_rows(d, od)
            worst = max(worst, float(rel.max()))
            # north_star: descriptors within 1e-4 relative.  The fp32 oracle is itself only an approximation of the
            # network: a few descriptors are ill-conditioned (attention pooling with a near-zero pooled vector before the
            # L2 normalisation).  So (1) 99.9 % within 1e-4 and nothing beyond 5e-4 against the oracle, and (2) against the
            # float64 evaluation of the same network on the same inputs (oracle.desc_fp64), on the worst rows and a strided
            # sample: every offender is a descriptor where the fp32 ORACLE is as far from the truth as the GPU path (GPU error
            # <= 1.5x oracle error + 2e-5), and every other row is within 1e-4 of the fp64 descriptor.
            assert (rel < 1e-4).mean() >= 0.999 and rel.max() < 5e-4, \
                f"{name} scale {i} {key}: descriptor rel err max {rel.max()}, within 1e-4: {(rel < 1e-4).mean()}"
            sel = np.unique(np.concatenate([np.argsort(rel)[-8:], np.arange(0, len(rel), max(1, len(rel) // 24))]))
            t64 = oracle.desc_fp64(osc[key]["feat"][torch.from_numpy(sel)], sd).numpy()
            e_gpu, e_orc = _rel_rows(d[sel].astype(np.float64), t64), _rel_rows(od[sel].astype(np.float64), t64)
            off = rel[sel] >= 1e-4                       # the offenders: wherever GPU and oracle disagree beyond 1e-4 ...
            bad = off & (e_gpu > 1.5 * e_orc + 2e-5)     # ... the fp32 oracle itself is that far from the truth
            assert not bad.any(), f"{name} scale {i} {key}: GPU vs fp64 {e_gpu[bad]} against oracle vs fp64 {e_orc[bad]}"
            # and everywhere else the GPU is within north_star's 1e-4 of the TRUE (fp64) descriptor, typically 100x closer
            assert (e_gpu[~off] < 1e-4).all() and np.median(e_gpu) < 2e-5, f"{name} scale {i} {key}: GPU vs fp64 max {e_gpu[~off].max()}"
        M, oM = int(sc["dM"].item()), len(osc["s_mids"])
        gs = set(zip(sc["s_mids"][:M].cpu().numpy().tolist(), sc["t_mids"][:M].cpu().numpy().tolist()))
        es = set(zip(osc["s_mids"].tolist(), osc["t_mids"].tolist()))
        rep[f"M{i}"] = (M, oM, len(gs ^ es))
        # arg-min flips between near-tied descriptors are possible at 1e-7 differences; allow a handful
        assert len(gs ^ es) <= max(2, oM // 200), f"{name} scale {i}: match sets differ by {len(gs ^ es)}"
    assert su == o_su and abs(nmut - o_nmut) <= max(2, o_nmut // 200)
    rre, rte = compute_rre(pose, o_pose), compute_rte(pose, o_pose)
    identical = all(a == b and x == 0 for a, b, x in rep.values())
    if identical:
        # identical match lists -> identical consensus set and RANSAC outcome, pose to rounding
        assert nind == o_nind and ninl == o_ninl
        assert rre < 0.1 and rte < 0.005, f"{name}: identical match lists but pose differs (RRE {rre}, RTE {rte})"
    # north_star: final (R,t) within the reference's own RRE/RTE success threshold of the oracle's (test.py:168-172),
    # whatever happened to individual arg-mins.  Only a pair without a consensus (both sides < 3 RANSAC correspondences or
    # no inliers: identity / arbitrary pose by construction) is exempt.
    if min(ninl, o_ninl) >= 3:
        assert rre < cfg.test.rre_thresh and rte < cfg.test.rte_thresh, \
            f"{name}: pose differs from the oracle's beyond the dataset thresholds (RRE {rre}, RTE {rte}; matches {rep})"
    else:
        assert max(ninl, o_ninl) < 3 or identical
    print(f"[{name}] matches {rep} inliers {ninl}/{o_ninl} consensus {nind}/{o_nind} RRE {rre:.4f} RTE {rte:.5f} worst desc rel {worst:.2e}")
    return pose, o_pose, rep


def test_pair_c1_against_oracle_and_golden(dev, oracle, c1):
    model = c1["model"].to(dev)
    pose, o_pose, rep = _compare_pair(model, c1["sd"], c1["cfg"], c1["data"], c1["perms"], oracle, "C1")
    g = np.load(os.path.join(ROOT, "tests", "golden", "c1_seed0.npz"))
    dbg = model.last_debug
    assert (dbg["fps_idx"][0].cpu().numpy() == g["s_fps"]).all()
    d, od = dbg["scales"][0]["s"]["desc"].cpu().numpy(), g["s0_src_desc"]
    den = np.abs(od).max(1)
    assert (np.abs(d - od).max(1) / np.where(den > 0, den, 1)).max() < 1e-4      # descriptors: 1e-4 rel (north_star)
    model.cpu()


def test_pair_c1_three_scales_outdoor_flags(dev, oracle):
    """3 scales, aligned-to-z (outdoor flags), no refinement, confidence 1.0 on the small cloud."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg("C3")
    cfg.patch.num_fps, cfg.patch.num_points_radius_estimate, cfg.match.iter_n = 200, 400, 4000
    model = init_synthetic_weights(bx.BufferX(cfg), seed=7)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    data = make_pair("C1", 5)
    data["is_aligned_to_global_z"] = True
    perms = oracle.draw_perms(cfg, 5000, 5000, 3)
    _compare_pair(model.to(dev), sd, cfg, data, perms, oracle, "C1x3")


def test_batched_descriptor_pass_equals_per_scale_pass(dev, oracle):
    """Without early exit the production path describes all 2*S (cloud, scale) sets in one batched pass
    (MiniSpinNet.forward_multi); the debug path runs them one by one.  Same kernels per patch -> identical results."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg("C2")
    cfg.patch.num_fps, cfg.patch.num_points_radius_estimate, cfg.match.iter_n = 300, 400, 5000
    assert cfg.match.get("enable_early_exit", True) is False
    model = init_synthetic_weights(bx.BufferX(cfg), seed=11).to(dev)
    data = make_pair("C1", 2)
    perms = oracle.draw_perms(cfg, 5000, 5000, 2)
    with torch.no_grad():
        a = model(data, perms=perms, ransac_seed=3, debug=False)         # batched
        b = model(data, perms=perms, ransac_seed=3, debug=True)          # per scale
        jobs = []
        dbg = model.last_debug
        for i in range(cfg.patch.num_scales):
            for j, key in ((0, "src_fds_pcd"), (1, "tgt_fds_pcd")):
                jobs.append((cu(data[key], dev), dbg["kpts"][j, :cfg.patch.num_fps].contiguous(), dbg["des_r"][i:i + 1],
                             cu(perms[i][j], dev, torch.int32)))
        outs = model.Desc.forward_multi(jobs, bool(data["is_aligned_to_global_z"]))
    assert np.array_equal(a[0], b[0]) and a[2:] == b[2:]                 # pose, inlier counts, scales used
    for i, sc in enumerate(dbg["scales"]):
        for j, side in ((0, "s"), (1, "t")):
            o = outs[2 * i + j]
            assert (o["desc"] == sc[side]["desc"]).all() and (o["equi"] == sc[side]["equi"]).all() and (o["R"] == sc[side]["R"]).all()
    model.cpu()


def test_c2_pair_registers_with_fitted_costnet(dev):
    """With the CostNet fitted on disjoint synthetic pairs (tests/tools/train_costnet.py) the C2 pairs register: the
    GPU pose meets the reference's 3DMatch success criterion (RRE < 15 deg, RTE < 0.3 m) against the ground truth."""
    import bufferx_b200 as bx
    from bufferx_b200.se3 import compute_rre, compute_rte
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg("C2")
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True).to(dev)
    for seed in (0, 3):
        data = make_pair("C2", seed)
        np.random.seed(seed)
        with torch.no_grad():
            pose, _, ninl, nmut, nind, su = model(data, ransac_seed=0)
        rre, rte = compute_rre(pose, data["relt_pose"]), compute_rte(pose, data["relt_pose"])
        assert rre < 15.0 and rte < 0.3, f"C2 seed {seed}: RRE {rre:.2f} deg RTE {rte:.3f} m (consensus {nind}, inliers {ninl})"
        assert nind >= 15
    model.cpu()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_c2_pairs_against_the_reference_forward(dev, oracle, seed):
    """The CUDA path against what the REFERENCE's own ``BufferX.forward`` produced (tests/golden/c2_seed*_reference.npz,
    written by oracle/ref_check.py in the build container: full C2 configuration, fitted CostNet, 21-52 RANSAC inliers,
    non-identity refined pose) and against the committed oracle fixture: same consensus set, same counts, final (R,t)
    within 0.1 deg / 5 mm of the reference's, >= 99.5 % of the reference's mutual matches."""
    import bufferx_b200 as bx
    from bufferx_b200.se3 import compute_rre, compute_rte
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg
    g = np.load(os.path.join(ROOT, "tests", "golden", f"c2_seed{seed}.npz"))
    r = np.load(os.path.join(ROOT, "tests", "golden", f"c2_seed{seed}_reference.npz"))
    cfg = workload_cfg("C2")
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True).to(dev)
    data = make_pair("C2", seed)
    perms = oracle.draw_perms(cfg, 20000, 20000, seed)
    with torch.no_grad():
        pose, _, ninl, nmut, nind, su = model(data, perms=perms, ransac_seed=0, debug=True)
    dbg = model.last_debug
    assert (dbg["fps_idx"][0].cpu().numpy() == g["s_fps"]).all() and (dbg["fps_idx"][1].cpu().numpy() == g["t_fps"]).all()
    assert np.allclose(dbg["des_r"].cpu().numpy().astype(np.float64), g["des_r"], atol=1e-6)
    common = total = 0
    stride = int(g["stride"])
    for i, sc in enumerate(dbg["scales"]):
        M = int(sc["dM"].item())
        gs = set(zip(sc["s_mids"][:M].cpu().numpy().tolist(), sc["t_mids"][:M].cpu().numpy().tolist()))
        rs = set(zip(r[f"s{i}_s_mids"].tolist(), r[f"s{i}_t_mids"].tolist()))
        common += len(gs & rs)
        total += len(rs)
        for side, key in (("s", "src"), ("t", "tgt")):
            rel = _rel_rows(sc[side]["desc"].cpu().numpy()[::stride], r[f"s{i}_{key}_desc"])
            assert (rel < 1e-4).mean() >= 0.99 and np.median(rel) < 2e-5     # vs the reference run itself (LRF-ulp voxel flips < 1 %)
    assert common >= 0.995 * total
    last = dbg["scales"][-1]
    inl = last["inlier_ind"][:int(last["dI"].item())].cpu().numpy()
    assert (inl == r["inlier_ind"]).all(), "consensus set differs from the reference run's"
    assert [ninl, nind, su] == [int(r["counts"][0]), int(r["counts"][2]), int(r["counts"][3])]
    assert abs(nmut - int(r["counts"][1])) <= 2
    assert np.abs(np.asarray(dbg["init_pose"]) - r["ransac_T"]).max() < 1e-6
    assert compute_rre(pose, r["pose"]) < 0.1 and compute_rte(pose, r["pose"]) < 0.005
    assert np.abs(r["pose"] - np.eye(4)).max() > 0.1 and ninl >= 20          # non-vacuous
    model.cpu()


def test_degenerate_pair_unrelated_clouds(dev, oracle):
    """Two unrelated clouds (a plane patch and a sphere shell, metres apart): a handful of mutual matches, a consensus
    set of at most one member, fewer than three RANSAC correspondences -> identity pose with 0 inliers, exactly like
    the oracle; nothing may crash on the empty / near-empty device-side lists."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, workload_cfg
    cfg = workload_cfg("C1")
    model = init_synthetic_weights(bx.BufferX(cfg))
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    rng = np.random.default_rng(5)
    src = np.c_[rng.uniform(-1, 1, (3000, 2)), rng.normal(0, 0.002, 3000)].astype(np.float32) + np.float32([5, 0, 0])
    v = rng.normal(size=(2500, 3))
    tgt = (v / np.linalg.norm(v, axis=1, keepdims=True) * 0.7).astype(np.float32) + np.float32([0, 4, 1])
    data = dict(src_fds_pcd=src, tgt_fds_pcd=tgt, relt_pose=np.eye(4, dtype=np.float32), is_aligned_to_global_z=False)
    perms = oracle.draw_perms(cfg, len(src), len(tgt), 0)
    model = model.to(dev)
    pose, o_pose, rep = _compare_pair(model, sd, cfg, data, perms, oracle, "degenerate")
    with torch.no_grad():
        out = model(data, perms=perms, ransac_seed=0)
    assert out[2] == 0 and np.allclose(out[0], np.eye(4))            # no inliers, identity
    model.cpu()


@pytest.mark.parametrize("trained,expect_scales", [(True, 1), (False, 3)])
def test_early_exit_mode(dev, oracle, trained, expect_scales):
    """a16: cfg.match.enable_early_exit = True (reference BUFFERX.py:424-439).  With the fitted CostNet the first scale
    already yields >= early_exit_min_inliers RANSAC inliers and the pair stops after one scale; with the random CostNet
    it runs all three (4 inliers < 5).  Same decision, counts and pose as the oracle."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg("C2")
    cfg.match.enable_early_exit = True
    cfg.match.early_exit_min_inliers = 5      # the weak seeded descriptor gives ~27 inliers at the first scale (the reference's 50 needs a real checkpoint)
    cfg.match.iter_n = 20000
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=trained)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    data = make_pair("C2", 3)
    perms = oracle.draw_perms(cfg, 20000, 20000, 3)
    model = model.to(dev)
    with torch.no_grad():
        pose, _, ninl, nmut, nind, su = model(data, perms=perms, ransac_seed=0)
    o_pose, o_ninl, o_nmut, o_nind, o_su, _ = oracle.register_pair(sd, cfg, data, perms, 0)
    assert su == o_su == expect_scales
    assert abs(nmut - o_nmut) <= max(2, o_nmut // 200)
    if nmut == o_nmut:
        assert (ninl, nind) == (o_ninl, o_nind)
        from bufferx_b200.se3 import compute_rre, compute_rte
        assert compute_rre(pose, o_pose) < 0.1 and compute_rte(pose, o_pose) < 0.005
    model.cpu()


def test_forward_draws_host_permutations_like_the_reference(dev, oracle, c1):
    """Without explicit perms forward() must consume NumPy's global RNG exactly like the reference
    (one np.random.choice(N, N, replace=False) per Desc call, src then tgt, per scale)."""
    model = c1["model"].to(dev)
    np.random.seed(0)
    with torch.no_grad():
        model(c1["data"], ransac_seed=0, debug=True)
    a = model.last_debug["scales"][0]["s"]["idx"].cpu().numpy()
    assert (a == c1["res"][5]["scales"][0]["src"]["idx"]).all()
    model.cpu()


# ------------------------------------------------------------------------------- full-size properties
def test_c2_full_size_pair(dev, oracle):
    """BASELINE config C2 (2x20000 points, 1500 key-points, 512 pts/patch, 3 scales, 50000 iters):
    whole pair against the oracle + size-independent properties."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg("C2")
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    data = make_pair("C2", 0)
    perms = oracle.draw_perms(cfg, 20000, 20000, 0)
    model = model.to(dev)
    _compare_pair(model, sd, cfg, data, perms, oracle, "C2")
    dbg = model.last_debug
    f = dbg["fps_idx"].cpu().numpy()
    assert f[0, 0] == 0 and len(set(f[0].tolist())) == f.shape[1]            # FPS: starts at 0, no repeats
    for si, sc in enumerate(dbg["scales"]):
        p = sc["s"]["raw_patches"].cpu().numpy()
        k = dbg["kpts"][0, :1500].cpu().numpy()
        assert (p[:, -1] == k).all()                                         # slot P-1 is the key-point
        d = np.linalg.norm(p - k[:, None], axis=-1)
        assert d.max() < float(dbg["des_r"][si].item()) + 1e-6                # every member is inside the ball
        idx = sc["s"]["idx"].cpu().numpy()
        inc = np.diff(idx, axis=1)
        assert ((inc > 0) | (idx[:, 1:] == idx[:, :1])).all()                # indices ascending, then first-hit padding
        e = sc["s"]["equi"].cpu().numpy()
        n = np.linalg.norm(e, axis=1)
        assert np.abs(n[n > 0] - 1).max() < 1e-5                              # equivariant maps are channel-normalised


def test_c3_kitti_sized_front_end(dev, oracle):
    """120000-point clouds: FPS (16-CTA cluster path), radius estimation and neighbour lists vs the oracle."""
    from bufferx_b200 import ops
    from bufferx_b200.synth import make_pair
    data = make_pair("C3", 0)
    src = data["src_fds_pcd"]
    idx, kp = ops.fps(cu(src, dev), [0, len(src)], 2048)
    eidx = oracle.fps(src, 2048)
    assert (idx[0].cpu().numpy() == eidx).all()
    kr = src[eidx[:2000]]
    r, m, _ = ops.radius_estimate(cu(kr, dev), cu(src, dev), [5, 2, 0.5])
    assert np.allclose(r.cpu().numpy(), np.array(oracle.radius_estimation(src[:1], kr[:1], src, kr, [5, 2, 0.5]), dtype=np.float32), atol=0)
    perm = np.random.RandomState(1).permutation(len(src)).astype(np.int32)
    pts4 = ops.permute_cloud(cu(src, dev), cu(perm, dev))
    q = src[eidx[:256]]
    pat, pidx = ops.select_patches(pts4, cu(q, dev), float(r[1].item()), 512, want_idx=True)
    eidx2, epat = oracle.select_patches(src, perm, q, float(r[1].item()), 512)
    assert (pidx.cpu().numpy() == eidx2).all() and (pat.cpu().numpy() == epat).all()


# ------------------------------------------------------------------------- conv kernels, layer by layer
def _torch_layer(geom, x, W, b, relu, kd, kh, kw):
    """torch-CPU statement of one conv layer (oracle-side arithmetic: F.conv3d / F.conv2d + explicit padding)."""
    import torch.nn.functional as F
    from oracle import oracle as O
    if geom == "cyl3d":
        y = F.conv3d(O._pad_cyl(x), W, b).squeeze(2)
    elif geom == "cyl2d":
        y = F.conv2d(O._pad_cyl(x), W, b)
    else:
        y = F.conv3d(x, W, b)
    return F.relu(y) if relu else y


@pytest.mark.parametrize("impl", ["sd", "tc"])
@pytest.mark.parametrize("geom,Cin,Cout,dims,k,n", [
    ("cyl3d", 16, 64, (3, 7, 20), (3, 3, 3), 37), ("cyl2d", 64, 128, (1, 7, 20), (1, 3, 3), 41),
    ("cyl2d", 128, 128, (1, 7, 20), (1, 3, 3), 19), ("cyl2d", 64, 32, (1, 7, 20), (1, 3, 3), 300),
    ("cyl2d", 32, 32, (1, 7, 20), (1, 3, 3), 5), ("valid3d", 32, 64, (18, 3, 18), (3, 3, 3), 9),
    ("valid3d", 64, 128, (14, 1, 14), (3, 1, 3), 13), ("valid3d", 32, 20, (2, 1, 2), (2, 1, 2), 77),
    ("cyl2d", 64, 64, (1, 7, 20), (1, 3, 3), 23), ("cyl2d", 128, 64, (1, 7, 20), (1, 3, 3), 7),
    ("valid3d", 128, 128, (12, 1, 12), (3, 1, 3), 11), ("valid3d", 64, 32, (6, 1, 6), (3, 1, 3), 50)])
def test_conv_layer_kernels(dev, geom, Cin, Cout, dims, k, n, impl):
    from bufferx_b200 import ops
    from bufferx_b200.models.patchnet import fold_conv_bn
    if impl == "sd" and geom == "valid3d" and (k != (3, 1, 3) or Cout % 16):
        pytest.skip("of the un-padded geometries the shifted-descriptor kernel serves the k = (3,1,3) layers")
    g = torch.Generator().manual_seed(Cin * 1000 + Cout + n)
    D, H, W_ = dims
    kd, kh, kw = k
    x = torch.randn((n, Cin, D, H, W_), generator=g)
    Wc = torch.randn((Cout, Cin, kd, kh, kw), generator=g) / (Cin * kd * kh * kw) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    relu = Cout != 20
    if geom == "cyl3d":
        ref = _torch_layer(geom, x, Wc, b, relu, kd, kh, kw)
    elif geom == "cyl2d":
        ref = _torch_layer(geom, x.squeeze(2), Wc.squeeze(2), b, relu, kd, kh, kw)
    else:
        ref = _torch_layer(geom, x, Wc, b, relu, kd, kh, kw)
    Wt, bf = fold_conv_bn(Wc, b)
    G = {"cyl3d": ops.GEOM_CYL3D, "cyl2d": ops.GEOM_CYL2D, "valid3d": ops.GEOM_VALID3D}[geom]
    OD, OH, OW = (1, 7, 20) if geom != "valid3d" else (D - kd + 1, H - kh + 1, W_ - kw + 1)
    xin = x.to(dev).reshape(n, Cin, -1).contiguous()
    if impl == "sd":                                                  # shifted-descriptor fp16-split kernel (production)
        out_cb = torch.full((n, Cout // 4, OD * OH * OW, 4), float("nan"), device=dev)
        flag = torch.zeros(1, dtype=torch.int32, device=dev)
        d_n = torch.tensor([n], dtype=torch.int32, device=dev) if geom == "valid3d" else None
        ops.conv_layer_sd(G, ops.to_blocked(xin), ops.conv_sd_weights(Wt.to(dev)), bf.to(dev), out_cb, n + (3 if geom == "valid3d" else 0), Cin, Cout, relu,
                          flag, d_n=d_n, D=D, W=W_)
        out = ops.from_blocked(out_cb)
        assert int(flag.item()) == 0
    else:                                                             # TF32 tensor-core kernel: channel-blocked activations
        out_cb = torch.full((n, Cout // 4, OD * OH * OW, 4), float("nan"), device=dev)
        ops.conv_layer_tc(G, ops.to_blocked(xin), ops.conv_tc_weights(Wt.to(dev)), bf.to(dev), out_cb, n, Cin, Cout, D, H, W_,
                          kd, kh, kw, relu)
        out = ops.from_blocked(out_cb)
    got = out.cpu().numpy().reshape(ref.shape)
    err = np.abs(got - ref.numpy()).max() / np.abs(ref.numpy()).max()
    assert err < 2e-5, f"{impl} {geom} Cin={Cin} Cout={Cout}: rel err {err}"     # fp32-grade (fp16 / 3xTF32 split) vs torch fp32


def test_conv_sd_dynamic_tiles_same_bits(dev):
    """bx_conv_layer_sd with a device-side tile counter (dynamic scheduling of the persistent CTAs) writes exactly what the
    static stride writes, launch after launch (the kernel rewinds the counter itself), incl. a device-side sample count."""
    from bufferx_b200 import ops
    torch.manual_seed(5)
    n, Cin, Cout = 700, 64, 64
    x = ops.sd_pack(torch.relu(torch.randn(n, Cin, 7, 20, device=dev)))
    Wt = torch.randn(9, Cin, Cout, device=dev) * 0.05
    w, b = ops.conv_sd_weights(Wt), torch.randn(Cout, device=dev) * 0.1
    ref = ops.conv_layer_sd(ops.GEOM_CYL2D, x, w, b, ops.conv_sd_buffer(n, Cout, dev).zero_(), n, Cin, Cout, True, None)
    ctr = torch.zeros(2, dtype=torch.int32, device=dev)
    for _ in range(3):
        out = ops.conv_layer_sd(ops.GEOM_CYL2D, x, w, b, ops.conv_sd_buffer(n, Cout, dev).zero_(), n, Cin, Cout, True, None, tile_ctr=ctr)
        assert torch.equal(out.view(torch.int16), ref.view(torch.int16))
        assert ctr.tolist() == [0, 0]



@pytest.mark.parametrize("tap", list(range(9)))
def test_conv_sd_single_tap_shifts(dev, tap):
    """One non-zero 3x3 tap at a time: every tap is a shifted VIEW (descriptor start address + (22 dy + dx) * 16 B) of the same
    shared-memory image, including the wrap columns and the zero rows -- the output must be the input moved by that tap."""
    from bufferx_b200 import ops
    import torch.nn.functional as F
    from oracle import oracle as O
    g = torch.Generator().manual_seed(tap)
    n, Cin, Cout = 11, 32, 32
    x = torch.randn((n, Cin, 7, 20), generator=g)
    Wc = torch.zeros((Cout, Cin, 3, 3))
    Wc[:, :, tap // 3, tap % 3] = torch.randn((Cout, Cin), generator=g) / Cin ** 0.5
    b = torch.zeros(Cout)
    ref = F.conv2d(O._pad_cyl(x), Wc, b)
    Wt = Wc.reshape(Cout, Cin, 9).permute(2, 1, 0).contiguous()
    out_cb = torch.full((n, Cout // 4, 140, 4), float("nan"), device=dev)
    ops.conv_layer_sd(ops.GEOM_CYL2D, ops.to_blocked(x.to(dev).reshape(n, Cin, -1).contiguous()), ops.conv_sd_weights(Wt.to(dev)), b.to(dev),
                      out_cb, n, Cin, Cout, False, None)
    got = ops.from_blocked(out_cb).cpu().numpy().reshape(ref.shape)
    err = np.abs(got - ref.numpy()).max() / np.abs(ref.numpy()).max()
    assert err < 2e-5, f"tap {tap} (dy {tap // 3}, dx {tap % 3}): rel err {err}"


@pytest.mark.parametrize("Cin,Cout,n", [(64, 128, 23), (128, 64, 9), (32, 32, 301), (64, 64, 1)])
def test_conv_sd_presplit_formats(dev, Cin, Cout, n):
    """The layer-to-layer format (fp16 hi/lo images over the padded 8 x 22 raster, written by the producing layer's epilogue
    and read back with bulk copies): presplit-in -> fp32-out, fp32-in -> presplit-out (values, zero rows, wrap columns) and a
    presplit -> presplit -> fp32 chain against torch fp32."""
    from bufferx_b200 import ops
    import torch.nn.functional as F
    from oracle import oracle as O
    g = torch.Generator().manual_seed(Cin + Cout + n)
    x = torch.randn((n, Cin, 7, 20), generator=g)
    W1 = torch.randn((Cout, Cin, 3, 3), generator=g) / (Cin * 9) ** 0.5
    b1 = torch.randn(Cout, generator=g) * 0.1
    W2 = torch.randn((Cin, Cout, 3, 3), generator=g) / (Cout * 9) ** 0.5
    b2 = torch.randn(Cin, generator=g) * 0.1
    y1 = F.relu(F.conv2d(O._pad_cyl(x), W1, b1))
    y2 = F.conv2d(O._pad_cyl(y1), W2, b2)
    wt = lambda W: ops.conv_sd_weights(W.reshape(W.shape[0], W.shape[1], 9).permute(2, 1, 0).contiguous().to(dev))
    xd = x.to(dev)
    rel = lambda a, b: float((a.cpu() - b).abs().max() / b.abs().max())
    # (a) presplit in -> fp32 out
    o = torch.full((n, Cout // 4, 140, 4), float("nan"), device=dev)
    ops.conv_layer_sd(ops.GEOM_CYL2D, ops.sd_pack(xd), wt(W1), b1.to(dev), o, n, Cin, Cout, True)
    assert rel(ops.from_blocked(o).view(n, Cout, 7, 20), y1) < 2e-5
    # (b) fp32 in -> presplit out: values + padding structure
    img = ops.conv_sd_buffer(n, Cout, dev)
    img.fill_(float("nan"))
    ops.conv_layer_sd(ops.GEOM_CYL2D, ops.to_blocked(xd.reshape(n, Cin, 140)), wt(W1), b1.to(dev), img, n, Cin, Cout, True)
    val, xp = ops.sd_unpack(img, n)
    assert rel(val, y1) < 2e-5
    assert (xp[:, :, 0] == 0).all(), "zero rows"
    assert (xp[:, :, 1:, 0] == xp[:, :, 1:, 20]).all() and (xp[:, :, 1:, 21] == xp[:, :, 1:, 1]).all(), "wrap columns"
    tail = img.view(Cout // 16, 2, 2, -1, 8)[:, :, :, n * 176:n * 176 + 22].float()
    assert (tail == 0).all(), "zero row after the last sample"
    # (c) presplit -> presplit -> fp32
    o2 = torch.full((n, Cin // 4, 140, 4), float("nan"), device=dev)
    ops.conv_layer_sd(ops.GEOM_CYL2D, img, wt(W2), b2.to(dev), o2, n, Cout, Cin, False)
    assert rel(ops.from_blocked(o2).view(n, Cin, 7, 20), y2) < 3e-5


def test_conv_sd_valid_raster_chain(dev):
    """CostNet's k = (3,1,3) layers on the shifted-descriptor kernel: un-padded D x W rasters, a device-side sample count
    below the capacity, presplit activations between the layers (16x16 -> 14x14 -> 12x12)."""
    from bufferx_b200 import ops
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(5)
    n, cap = 37, 50
    x = torch.randn((n, 64, 16, 1, 16), generator=g)
    W1 = torch.randn((64, 64, 3, 1, 3), generator=g) / (64 * 9) ** 0.5
    W2 = torch.randn((128, 64, 3, 1, 3), generator=g) / (64 * 9) ** 0.5
    b1, b2 = torch.randn(64, generator=g) * 0.1, torch.randn(128, generator=g) * 0.1
    y1 = F.relu(F.conv3d(x, W1, b1))
    y2 = F.relu(F.conv3d(y1, W2, b2))
    wt = lambda W: ops.conv_sd_weights(W.reshape(W.shape[0], W.shape[1], 9).permute(2, 1, 0).contiguous().to(dev))
    d_n = torch.tensor([n], dtype=torch.int32, device=dev)
    xin = torch.zeros((cap, 16, 256, 4), device=dev)
    xin[:n] = ops.to_blocked(x.to(dev).reshape(n, 64, 256))
    mid = ops.conv_sd_buffer(cap, 64, dev, 14 * 14)
    mid.fill_(float("nan"))
    ops.conv_layer_sd(ops.GEOM_VALID3D, xin, wt(W1), b1.to(dev), mid, cap, 64, 64, True, None, d_n=d_n, D=16, W=16)
    out = torch.full((cap, 32, 144, 4), float("nan"), device=dev)
    ops.conv_layer_sd(ops.GEOM_VALID3D, mid, wt(W2), b2.to(dev), out, cap, 64, 128, True, None, d_n=d_n, D=14, W=14)
    got = ops.from_blocked(out[:n]).view(n, 128, 12, 1, 12).cpu()
    assert float((got - y2).abs().max() / y2.abs().max()) < 3e-5
    assert torch.isnan(out[n:]).all()                 # samples beyond the device-side count are not touched


def test_conv_sd_fp16_range_flag_and_fallback(dev):
    """An activation beyond fp16 range cannot be split into fp16 operands: the kernel raises the sticky flag (and the model
    then re-runs on the TF32 kernel, BufferX._decode)."""
    from bufferx_b200 import ops
    n, Cin, Cout = 3, 16, 32
    x = torch.ones((n, Cin, 140), device=dev)
    x[1, 3, 17] = 1.0e5
    Wt = torch.full((9, Cin, Cout), 0.01, device=dev)
    out = torch.empty((n, Cout // 4, 140, 4), device=dev)
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    ops.conv_layer_sd(ops.GEOM_CYL2D, ops.to_blocked(x), ops.conv_sd_weights(Wt), torch.zeros(Cout, device=dev), out, n, Cin, Cout, True, flag)
    assert int(flag.item()) == 1
    x[1, 3, 17] = 2.0
    flag.zero_()
    ops.conv_layer_sd(ops.GEOM_CYL2D, ops.to_blocked(x), ops.conv_sd_weights(Wt), torch.zeros(Cout, device=dev), out, n, Cin, Cout, True, flag)
    assert int(flag.item()) == 0
    # an OUTPUT beyond fp16 range cannot be written in the presplit format either
    big = torch.full((9, Cin, Cout), 500.0, device=dev)
    ops.conv_layer_sd(ops.GEOM_CYL2D, ops.to_blocked(x), ops.conv_sd_weights(big), torch.zeros(Cout, device=dev), ops.conv_sd_buffer(n, Cout, dev), n, Cin, Cout, True, flag)
    assert int(flag.item()) == 1


# ------------------------------------------------------------------------------ graphs / async pairs
def test_cuda_graph_replay_and_async_pairs_match_eager(dev, oracle, c1):
    """Captured-graph replays on two slot streams (pairs in flight) return exactly the eager results."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import make_pair
    model = c1["model"].to(dev)
    cfg = c1["cfg"]
    pairs = [make_pair("C1", s) for s in range(4)]
    perms = [oracle.draw_perms(cfg, 5000, 5000, 10 + s) for s in range(4)]
    model.enable_cuda_graphs(False)
    with torch.no_grad():
        eager = [model(p, perms=q) for p, q in zip(pairs, perms)]
        model.enable_cuda_graphs(True, slots_per_shape=2)
        outs, handles = [], []
        for p, q in zip(pairs, perms):
            if len(handles) == 2:
                outs.append(handles.pop(0).result())
            handles.append(model.forward_async(p, perms=q))
        outs += [h.result() for h in handles]
        again = model(pairs[0], perms=perms[0])              # forward() itself replays the graph when enabled
    model.enable_cuda_graphs(False)
    for e, o in zip(eager, outs):
        assert np.array_equal(np.asarray(e[0]), np.asarray(o[0])) and e[2:] == o[2:]
    assert np.array_equal(np.asarray(eager[0][0]), np.asarray(again[0])) and eager[0][2:] == again[2:]
    model.cpu()


# ------------------------------------------------------------------------------ other BASELINE configs
def test_c3_kitti_sized_pair(dev, oracle):
    """BASELINE config C3 (2x120000 points, 2048 key-points, aligned-to-z, confidence 1.0, no refinement);
    RANSAC iterations reduced for the CPU oracle's sake -- the GPU side runs the same count."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg("C3")
    cfg.match.iter_n = 5000
    model = init_synthetic_weights(bx.BufferX(cfg))
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    data = make_pair("C3", 1)
    perms = oracle.draw_perms(cfg, 120000, 120000, 1)
    _compare_pair(model.to(dev), sd, cfg, data, perms, oracle, "C3")


def test_c5_heterogeneous_pair(dev, oracle):
    """BASELINE config C5 (60000-point vs 30000-point clouds of one scene, outdoor flags)."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg("C5")
    cfg.match.iter_n = 5000
    cfg.patch.num_fps = 600
    model = init_synthetic_weights(bx.BufferX(cfg))
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    data = make_pair("C5", 0)
    perms = oracle.draw_perms(cfg, 60000, 30000, 2)
    _compare_pair(model.to(dev), sd, cfg, data, perms, oracle, "C5")


# ----------------------------------------------------------------------------------------- a17 / a18
@pytest.mark.parametrize("radius,qb,sb", [(0.35, [300, 200], [3500, 2500]), (0.15, [777], [9000]), (0.9, [64, 64], [2000, 1000])])
def test_radius_neighbors_bit_exact(dev, oracle, radius, qb, sb):
    from bufferx_b200 import ops
    rng = np.random.default_rng(int(radius * 100))
    s = rng.uniform(-2, 2, (sum(sb), 3)).astype(np.float32)
    q = (s[rng.choice(len(s), sum(qb), replace=False)] + rng.normal(scale=0.01, size=(sum(qb), 3))).astype(np.float32)
    got = ops.radius_neighbors(cu(q, dev), cu(s, dev), qb, sb, radius).cpu().numpy()
    exp = oracle.radius_neighbors(q, s, qb, sb, radius)
    assert got.shape == exp.shape and (got == exp).all()


def test_grid_subsample_matches_oracle(dev, oracle):
    from bufferx_b200 import ops
    rng = np.random.default_rng(4)
    pts = (rng.uniform(-3, 3, (50000, 3)) * [1, 1, 0.4]).astype(np.float32)
    for dl in (0.1, 0.35):
        keys, xyz, cnt = ops.grid_subsample(cu(pts, dev), dl)
        ek, exyz, ecnt = oracle.grid_subsample(pts, dl)
        k = keys.cpu().numpy().astype(np.uint64)
        o = np.argsort(k)
        assert (k[o] == ek).all() and (cnt.cpu().numpy()[o] == ecnt).all()             # cell ids and counts: bit-exact
        assert np.abs(xyz.cpu().numpy()[o] - exyz).max() < 2e-6                         # barycentres: fp32 summation order


# ------------------------------------------------------------------ SURVEY 8(f) row 1: geometric bootstrapping
@pytest.mark.gpu
@pytest.mark.parametrize("name,ns,nt", [("C1", 5000, 5000), ("C3", 30000, 24000), ("C5", 20000, 9000)])
def test_sphericity_based_voxel_analysis(dev, oracle, name, ns, nt):
    """GPU PCA / z-range against the float64 oracle (itself pinned against sklearn): variances 1e-9 rel, components
    1e-8, identical (voxel_size, is_aligned_to_global_z), sphericity 1e-9."""
    from bufferx_b200 import ops
    from bufferx_b200.synth import make_pair
    from bufferx_b200.bootstrap import sphericity_based_voxel_analysis
    data = make_pair(name, 2, n_src=ns, n_tgt=nt)
    src, tgt = data["src_fds_pcd"], data["tgt_fds_pcd"]
    st = np.random.RandomState(7)
    i_s = st.choice(ns, size=ns // 10, replace=False)
    i_t = st.choice(nt, size=nt // 10, replace=False)
    mean, var, comps = ops.pca_analysis(cu(src, dev), cu(i_s.astype(np.int32), dev, torch.int32))
    _, _, o_mean, o_var, o_comps = oracle.pca_alignment(src, i_s)
    assert np.allclose(mean.cpu().numpy(), o_mean, atol=1e-10)
    assert np.allclose(var.cpu().numpy(), o_var, rtol=1e-9)
    assert np.allclose(comps.cpu().numpy(), o_comps, atol=1e-8)
    got = sphericity_based_voxel_analysis(src, tgt, i_s, i_t, device=dev)
    exp = oracle.sphericity_based_voxel_analysis(src, tgt, i_s, i_t)
    assert got[0] == exp[0] and got[2] == exp[2] and abs(got[1] - exp[1]) < 1e-9 * max(1.0, abs(exp[1]))


@pytest.mark.gpu
@pytest.mark.parametrize("n,voxel", [(5000, 0.035), (60000, 0.3), (1, 0.5), (777, 10.0)])
def test_voxel_down_sample(dev, oracle, n, voxel):
    """Same occupied voxels and counts as the oracle (exact), means within 1e-6 (fp64 sums, fp32 output)."""
    from bufferx_b200 import ops
    rng = np.random.default_rng(n)
    pts = (rng.normal(size=(n, 3)) * np.array([8.0, 5.0, 1.5])).astype(np.float32)
    keys, xyz, cnt = ops.voxel_down_sample(cu(pts, dev), voxel)
    order = torch.argsort(keys)
    k, x, c = keys[order].cpu().numpy(), xyz[order].cpu().numpy(), cnt[order].cpu().numpy()
    ek, em, ec = oracle.voxel_down_sample(pts, voxel)
    assert (k == ek).all() and (c == ec).all()
    assert np.abs(x - em).max() <= 1e-6 * max(1.0, np.abs(em).max())
