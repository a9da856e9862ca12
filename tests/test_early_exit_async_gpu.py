"""Early exit on the throughput path: forward_async and captured graphs with cfg.match.enable_early_exit, the decision taken
on the device (bx_early_exit_gate) and the later scales' work sized by device-side key-point counts.

Checks the count contract of every descriptor kernel that takes one, the gate against PoseEstimator.compute_confidence_score,
bit-identity of exiting / non-exiting pairs with the early-exit-off flow on the same inputs, agreement with the oracle, graph
replay across both outcomes, the NumPy RNG rule of forward_async and the fp16-range fall-back."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

NAN = float("nan")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


def i32(v, dev):
    return torch.tensor([v], dtype=torch.int32, device=dev)


def _cloud(rng, n, dev):
    return torch.from_numpy(rng.uniform(-1, 1, (n, 3)).astype(np.float32)).to(dev)


# ------------------------------------------------------------------------------------------ 1. count contract
@pytest.mark.parametrize("n_pts", [3000, 15000])     # below / above ops.GRID_MIN_POINTS: streaming scan / hash grid
def test_select_patches_counts(dev, n_pts):
    from bufferx_b200 import ops
    rng = np.random.default_rng(n_pts)
    K, P, k = 40, 64, 17
    grid = n_pts >= ops.GRID_MIN_POINTS
    jobs = []
    for j in range(2):
        pts = _cloud(rng, n_pts, dev)
        pts4 = ops.permute_cloud(pts, torch.arange(n_pts, dtype=torch.int32, device=dev))
        jobs.append((pts4, pts[torch.randperm(n_pts, device=dev)[:K]].contiguous(), torch.tensor([0.3 + 0.1 * j], device=dev)))
    for c in (0, k, K):
        ref = torch.empty((2 * c, P, 3), device=dev)
        if c:
            ops.select_patches_batched([(p, kp[:c].contiguous(), r) for p, kp, r in jobs], P, ref, grid=grid)
        got = torch.full((2 * K, P, 3), NAN, device=dev)
        ops.select_patches_batched(jobs, P, got, grid=grid, d_K=[i32(c, dev)] * 2)
        for j in range(2):
            assert torch.equal(got[j * K:j * K + c], ref[j * c:(j + 1) * c])
            assert torch.isnan(got[j * K + c:(j + 1) * K]).all()


def test_lrf_counts(dev):
    from bufferx_b200 import ops
    rng = np.random.default_rng(2)
    G, R, P, k = 2, 24, 64, 9
    patches = torch.from_numpy(rng.normal(0, 0.2, (G * R, P, 3)).astype(np.float32)).to(dev)
    radii = torch.tensor([0.4, 0.7], device=dev)
    for aligned in (False, True):
        for c in (0, k, R):
            d, Rt, ra = (torch.full(s, NAN, device=dev) for s in ((G * R, P, 3), (G * R, 3, 3), (G * R, 3)))
            ops.lrf(patches, radii, aligned, delta=d, Rt=Rt, ra=ra, r_group=R, d_K=torch.tensor([c] * G, dtype=torch.int32, device=dev))
            for g in range(G):
                rows = slice(g * R, g * R + c)
                if c:
                    ed, eR, ea = ops.lrf(patches[rows].contiguous(), radii[g:g + 1], aligned)
                    assert torch.equal(d[rows], ed) and torch.equal(Rt[rows], eR) and torch.equal(ra[rows], ea)
                tail = slice(g * R + c, (g + 1) * R)
                assert torch.isnan(d[tail]).all() and torch.isnan(Rt[tail]).all() and torch.isnan(ra[tail]).all()


@pytest.fixture(scope="module")
def desc_inputs(dev):
    """Normalised patches of a C2 cloud and the seeded descriptor network."""
    import bufferx_b200 as bx
    from bufferx_b200 import ops
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg("C2")
    model = init_synthetic_weights(bx.BufferX(cfg)).to(dev).eval()
    data = make_pair("C2", 0)
    pts = torch.from_numpy(data["src_fds_pcd"]).to(dev).contiguous()
    K = 24
    pts4 = ops.permute_cloud(pts, torch.arange(pts.shape[0], dtype=torch.int32, device=dev))
    kp = pts[torch.arange(K, device=dev) * 700].contiguous()
    patches, _ = ops.select_patches(pts4, kp, 0.35, cfg.patch.num_points_per_patch)
    delta, _, _ = ops.lrf(patches, 0.35, False)
    return dict(model=model, delta=delta, K=K)


def _spt(model, delta):
    from bufferx_b200 import ops
    net = model.Desc
    prep = net.prepared(delta.device)
    return ops.spt_pnt_sd(delta, prep["voxels"], prep["rot"], net.delta / net.rad_n, net.voxel_sample, prep["w_pnt"], prep["b_pnt"], net.azi_n)


def test_spt_pnt_sd_counts(dev, desc_inputs):
    from bufferx_b200 import ops
    model, delta, K = desc_inputs["model"], desc_inputs["delta"], desc_inputs["K"]
    net = model.Desc
    prep = net.prepared(dev)
    for c in (0, 7, K):
        feat = ops.conv_sd_buffer(K, 48, dev)        # NaN-filled, then written through the C-ABI with the count
        feat.fill_(NAN)
        lib = ops.load_library()
        ops._check(lib.bx_spt_pnt_sd_n(ops._dp(delta), K, delta.shape[1], ops._dp(prep["voxels"]), prep["voxels"].shape[0], net.azi_n,
                                       ops._dp(prep["rot"]), float(net.delta / net.rad_n), net.voxel_sample, ops._dp(prep["w_pnt"]),
                                       ops._dp(prep["b_pnt"]), ops._dp(feat), feat.shape[2], None, ops._dp(i32(c, dev)), ops._stream()), "spt")
        val, pad = ops.sd_unpack(feat, K)
        if c:
            ref = _spt(model, delta[:c].contiguous())
            rval, rpad = ops.sd_unpack(ref, c)
            assert torch.equal(pad[:c], rpad)                                   # values, wrap columns and zero rows
            if c < K:
                assert (pad[c, :, 0] == 0).all()                                # the zero row that follows sample c - 1
        assert torch.isnan(val[c:]).all()


@pytest.mark.parametrize("geom", ["CYL3D", "CYL2D"])
def test_conv_layer_sd_counts_cylindrical(dev, desc_inputs, geom):
    from bufferx_b200 import ops
    model, delta, K = desc_inputs["model"], desc_inputs["delta"], desc_inputs["K"]
    L = model.Desc.conv_net.folded()
    x = _spt(model, delta)                                                       # presplit input of K samples
    li = 0 if geom == "CYL3D" else 1
    if li == 1:
        y = ops.conv_sd_buffer(K, 64, dev)
        ops.conv_layer_sd(ops.GEOM_CYL3D, x, L[0]["w_sd"], L[0]["b"], y, K, 16, 64, True)
        x = y
    l = L[li]
    g = ops.GEOM_CYL3D if li == 0 else ops.GEOM_CYL2D
    for c in (0, 11, K):
        out = torch.full((K, l["cout"] // 4, 140, 4), NAN, device=dev)
        ops.conv_layer_sd(g, x, l["w_sd"], l["b"], out, K, l["cin"], l["cout"], l["relu"], d_n=i32(c, dev))
        if c:
            # the un-gated call on c samples reads an image laid out for c samples (its planes are conv_sd_rows(c) rows apart)
            xc = x[:, :, :ops.conv_sd_rows(c)].contiguous()
            ref = torch.empty((c, l["cout"] // 4, 140, 4), device=dev)
            ops.conv_layer_sd(g, xc, l["w_sd"], l["b"], ref, c, l["cin"], l["cout"], l["relu"])
            assert torch.equal(out[:c], ref)
        assert torch.isnan(out[c:]).all()


def test_pool_desc_counts(dev, desc_inputs):
    from bufferx_b200 import ops
    prep = desc_inputs["model"].Desc.prepared(dev)
    K = 30
    x = torch.randn((K, 8, 140, 4), device=dev).abs()
    for c in (0, 13, K):
        desc, equi = torch.full((K, 32), NAN, device=dev), torch.full((K, 32, 7, 20), NAN, device=dev)
        ops.pool_desc(x, prep["w1"], prep["b1"], prep["w2"], prep["b2"], desc=desc, equi=equi, channels_last=True, d_K=i32(c, dev))
        if c:
            rd, re = ops.pool_desc(x[:c].contiguous(), prep["w1"], prep["b1"], prep["w2"], prep["b2"], channels_last=True)
            assert torch.equal(desc[:c], rd) and torch.equal(equi[:c], re)
        assert torch.isnan(desc[c:]).all() and torch.isnan(equi[c:]).all()


def test_mutual_nn_counts(dev):
    from bufferx_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(4)
    K = 300
    a = torch.nn.functional.normalize(torch.randn((K, 32), generator=g), dim=1).to(dev)
    b = (a + 0.3 * torch.randn((K, 32), generator=g).to(dev))[torch.randperm(K, generator=g).to(dev)].contiguous()
    for ca, cb in ((0, K), (K, 0), (0, 0), (117, 117), (117, K), (K, 200), (K, K)):
        s = torch.full((K,), -7, dtype=torch.int32, device=dev)
        t, dM = s.clone(), i32(-7, dev)
        ops.mutual_nn(a, b, out=(s, t, dM), d_Ka=i32(ca, dev), d_Kb=i32(cb, dev))
        M = int(dM.item())
        if ca == 0 or cb == 0:
            assert M == 0 and (s == -7).all() and (t == -7).all()
            continue
        rs, rt, rM, _, _ = ops.mutual_nn(a[:ca].contiguous(), b[:cb].contiguous())
        assert M == int(rM.item()) > 0
        assert torch.equal(s[:M], rs[:M]) and torch.equal(t[:M], rt[:M]) and (s[M:] == -7).all()


# ------------------------------------------------------------------------------------------------ 2. gate
@pytest.mark.parametrize("S", [1, 3])
@pytest.mark.parametrize("delta_inl", [-1, 0, 1])
def test_early_exit_gate(dev, S, delta_inl):
    from bufferx_b200 import ops
    from bufferx_b200.models.pose_estimator import PoseEstimator
    from bufferx_b200.synth import workload_cfg
    cfg = workload_cfg("C2")
    cfg.match.early_exit_min_inliers = 5
    n_inl = 5 + delta_inl
    res = torch.zeros(18, dtype=torch.float64)
    res[16:18].view(torch.int32)[:] = torch.tensor([n_inl, 3, 100, 0], dtype=torch.int32)
    res = res.to(dev)
    caps = [1500, 3000, 3000 * (S - 1) + 1]
    counts = torch.full((3,), -1, dtype=torch.int32, device=dev)
    su = torch.zeros(1, dtype=torch.float64, device=dev)
    ops.early_exit_gate(res, 5, caps, counts, S, su)
    stop = PoseEstimator(cfg).compute_confidence_score(n_inl)
    assert stop == (delta_inl >= 0)
    assert counts.tolist() == ([0, 0, 0] if stop else caps)
    assert su.item() == (1.0 if stop else float(S))


# ------------------------------------------------------------------------------------------------ 3-9. pairs
def _cfg(exit=True, S=3, trained=True):
    from bufferx_b200.synth import workload_cfg
    cfg = workload_cfg("C2")
    cfg.match.enable_early_exit = exit
    cfg.match.early_exit_min_inliers = 5
    cfg.match.iter_n = 20000
    if S != cfg.patch.num_scales:
        cfg.patch.num_scales = S
        cfg.patch.search_radius_thresholds = list(cfg.patch.search_radius_thresholds)[:S]
    return cfg


def _model(cfg, sd, dev):
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights
    m = init_synthetic_weights(bx.BufferX(cfg))
    m.load_state_dict(sd)
    return m.to(dev).eval()


@pytest.fixture(scope="module")
def pairs(dev, oracle):
    """C2 seed 3 with explicit perms; fitted (exits) and random (runs every scale) CostNet state dicts."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, make_pair
    cfg = _cfg()
    sds = {t: {k: v.detach().clone() for k, v in init_synthetic_weights(bx.BufferX(cfg), trained_pose=t).state_dict().items()}
           for t in (True, False)}
    data = make_pair("C2", 3)
    perms = oracle.draw_perms(cfg, 20000, 20000, 3)
    return dict(cfg=cfg, sd=sds, data=data, perms=perms)


def _eq(a, b):
    return np.array_equal(np.asarray(a[0]), np.asarray(b[0])) and tuple(a[2:]) == tuple(b[2:])


@pytest.mark.parametrize("trained,expect_scales", [(True, 1), (False, 3)])
def test_async_early_exit_bit_identical_and_matches_oracle(dev, oracle, pairs, trained, expect_scales):
    """Exit: identical to the early-exit-off flow with one scale (its threshold, the scale-0 perms).  No exit: identical to
    the early-exit-off flow with every scale.  Both agree with the oracle like test_early_exit_mode."""
    sd, data, perms = pairs["sd"][trained], pairs["data"], pairs["perms"]
    with torch.no_grad():
        out = _model(_cfg(), sd, dev).forward_async(data, perms=perms).result()
        S_ref = 1 if expect_scales == 1 else 3
        ref = _model(_cfg(exit=False, S=S_ref), sd, dev).forward_async(data, perms=perms[:S_ref]).result()
    assert out[5] == expect_scales
    assert _eq(out, ref), (out[2:], ref[2:])
    o_pose, o_ninl, o_nmut, o_nind, o_su, _ = oracle.register_pair(sd, _cfg(), data, perms, 0)
    pose, _, ninl, nmut, nind, su = out
    assert su == o_su == expect_scales
    assert abs(nmut - o_nmut) <= max(2, o_nmut // 200)
    if nmut == o_nmut:
        from bufferx_b200.se3 import compute_rre, compute_rte
        assert (ninl, nind) == (o_ninl, o_nind)
        assert compute_rre(pose, o_pose) < 0.1 and compute_rte(pose, o_pose) < 0.005


def _unrelated(data):
    rng = np.random.default_rng(11)
    tgt = data["tgt_fds_pcd"]
    v = rng.normal(size=tgt.shape)
    tgt = (v / np.linalg.norm(v, axis=1, keepdims=True) * 0.7).astype(np.float32) + np.float32([0, 4, 1])
    return dict(data, tgt_fds_pcd=tgt)


def _degenerate():
    rng = np.random.default_rng(5)
    src = np.c_[rng.uniform(-1, 1, (3000, 2)), rng.normal(0, 0.002, 3000)].astype(np.float32) + np.float32([5, 0, 0])
    v = rng.normal(size=(2500, 3))
    tgt = (v / np.linalg.norm(v, axis=1, keepdims=True) * 0.7).astype(np.float32) + np.float32([0, 4, 1])
    return dict(src_fds_pcd=src, tgt_fds_pcd=tgt, relt_pose=np.eye(4, dtype=np.float32), is_aligned_to_global_z=False)


def test_graphs_replay_both_outcomes(dev, oracle, pairs):
    """Six pairs in flight on captured graphs, exiting and non-exiting pairs of one shape alternating so that every slot's
    graph is replayed for both outcomes, plus the unrelated-cloud pair of test_degenerate_pair_unrelated_clouds (another
    shape, a handful of inliers under this configuration); each result equals its eager
    forward_async result.  That the capture succeeds shows the path has no host synchronisation."""
    cfg = _cfg()
    model = _model(cfg, pairs["sd"][True], dev)
    exit_pair, stay_pair, degen = pairs["data"], _unrelated(pairs["data"]), _degenerate()
    perms = pairs["perms"]
    perms_d = oracle.draw_perms(cfg, 3000, 2500, 0)
    with torch.no_grad():
        eager = {name: model.forward_async(d, perms=p).result()
                 for name, d, p in (("exit", exit_pair, perms), ("stay", stay_pair, perms), ("degen", degen, perms_d))}
        assert eager["exit"][5] == 1 and eager["stay"][5] == 3
        model.enable_cuda_graphs(True, slots_per_shape=6)
        seq = ["exit", "stay"] * 3 + ["stay", "exit"] * 3 + ["degen"]     # launch i and i + 6 share a slot
        src = dict(exit=(exit_pair, perms), stay=(stay_pair, perms), degen=(degen, perms_d))
        handles, results = [], []
        for name in seq:
            if len(handles) == 6:
                n0, h0 = handles.pop(0)
                results.append((n0, h0.result()))
            handles.append((name, model.forward_async(src[name][0], perms=src[name][1])))
        results += [(n, h.result()) for n, h in handles]
        slots = model._slots[(20000, 20000, False, True, 5)]
        assert len(slots) == 6 and all(sl.graph is not None for sl in slots)
    model.enable_cuda_graphs(False)
    for name, r in results:
        assert _eq(r, eager[name]), (name, r[2:], eager[name][2:])
    assert {r[5] for n, r in results if n != "degen"} == {1, 3}


def test_threshold_change_recaptures(dev, pairs):
    cfg = _cfg()
    model = _model(cfg, pairs["sd"][True], dev)
    model.enable_cuda_graphs(True, slots_per_shape=1)
    with torch.no_grad():
        a = model.forward_async(pairs["data"], perms=pairs["perms"]).result()
        cfg.match.early_exit_min_inliers = 10 ** 6
        b = model.forward_async(pairs["data"], perms=pairs["perms"]).result()
    keys = set(model._slots)
    model.enable_cuda_graphs(False)
    assert a[5] == 1 and b[5] == 3
    assert {(20000, 20000, False, True, 5), (20000, 20000, False, True, 10 ** 6)} <= keys


def _draws(n_s, n_t, k):
    for _ in range(k):
        np.random.choice(n_s, n_s, replace=False)
        np.random.choice(n_t, n_t, replace=False)


def _state_eq(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


def test_rng_consumption(dev, pairs):
    """forward_async with early exit draws all 2*S permutations whether or not the pair exits; eager forward keeps the
    reference's order (an exiting pair draws two)."""
    cfg = _cfg()
    with torch.no_grad():
        for trained in (True, False):
            model = _model(cfg, pairs["sd"][trained], dev)
            np.random.seed(1)
            model.forward_async(pairs["data"]).result()
            after = np.random.get_state()
            np.random.seed(1)
            _draws(20000, 20000, 3)
            assert _state_eq(after, np.random.get_state())
        model = _model(cfg, pairs["sd"][True], dev)
        np.random.seed(1)
        out = model(pairs["data"], ransac_seed=0)
        after = np.random.get_state()
        np.random.seed(1)
        _draws(20000, 20000, 1)
    assert out[5] == 1 and _state_eq(after, np.random.get_state())


def test_forward_async_timing_still_refused(dev, pairs):
    from bufferx_b200 import ops
    cfg = _cfg()
    cfg.test.enable_timing = True
    model = _model(cfg, pairs["sd"][True], dev)
    with pytest.raises(ops.BufferXError):
        model.forward_async(pairs["data"], perms=pairs["perms"])


def test_fp16_fallback_with_early_exit(dev, pairs):
    """Point layer scaled so that features leave fp16 range: forward_async with early exit returns what eager forward
    returns with the same perms after its own switch to the TF32 kernels."""
    sd = {k: v.clone() for k, v in pairs["sd"][True].items()}
    for k in ("pnt_layer.0.weight", "pnt_layer.0.bias", "pnt_layer.1.running_mean", "pnt_layer.1.bias"):
        sd["Desc." + k] = sd["Desc." + k] * 1.0e6
    with torch.no_grad():
        m1 = _model(_cfg(), sd, dev)
        got = m1.forward_async(pairs["data"], perms=pairs["perms"]).result()
        assert m1.Desc.conv_net.force_tf32
        m2 = _model(_cfg(), sd, dev)
        exp = m2(pairs["data"], perms=pairs["perms"])
        assert m2.Desc.conv_net.force_tf32
    assert _eq(got, exp)
