"""Size classes on the throughput path: one captured graph per (C_src, C_tgt, aligned) capacity serves every pair whose
clouds fit, the true point counts read on the device by FPS, the radius histogram, the cloud permutation and both patch
gatherers.

Checks the count contract of each of those kernels with POISONED padding (rows beyond the count hold points that would
change the result if they were read), then the model: pairs of many sizes on class graphs against eager forward, with and
without early exit, aligned clouds in two different classes, the DataParallel drop-in loop, inputs from another stream or
pinned memory, and the fp16-range fall-back."""
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
    return torch.tensor(v if isinstance(v, list) else [v], dtype=torch.int32, device=dev)


def _lattice(rng, n):
    """Points of a coarse integer lattice, many of them duplicated: FPS meets exact distance ties at every step."""
    base = rng.integers(-6, 7, size=(max(n // 3, 1), 3)).astype(np.float32) * np.float32(0.25)
    pts = base[rng.integers(0, base.shape[0], size=n)]
    pts[0] = (0.5, 0.25, -0.75)
    return pts


# ------------------------------------------------------------------------------------------ 1. count contract
@pytest.mark.parametrize("cap,sizes", [(4096, [255, 256, 257, 511, 512, 513, 3000]), (16384, [8193, 9000, 16383, 16384])])
def test_fps_counts(dev, oracle, cap, sizes):
    """Capacity buffers with one far point right behind the cloud (it would win step 1); N at 2^k - 1, 2^k, 2^k + 1 inside
    one class so that the tie rule's block size changes.  Same indices and key-points as ops.fps on the exact cloud and as
    the oracle."""
    from bufferx_b200 import ops
    rng = np.random.default_rng(cap)
    npoint = 200
    for a, b in zip(sizes[0::2], sizes[1::2] + sizes[:1]):
        clouds = [_lattice(rng, a), _lattice(rng, b)]
        buf = np.full((2 * cap, 3), 40.0, dtype=np.float32)             # poison: far outside the lattice
        buf[:a], buf[cap:cap + b] = clouds
        xyz = torch.from_numpy(buf).to(dev)
        idx, kp = ops.fps(xyz, [0, cap, 2 * cap], npoint, d_counts=i32([a, b], dev))
        for c, cl in enumerate(clouds):
            e_idx, e_kp = ops.fps(torch.from_numpy(cl).to(dev), [0, cl.shape[0]], npoint)
            assert torch.equal(idx[c], e_idx[0]) and torch.equal(kp[c], e_kp[0]), (cap, cl.shape[0])
            assert np.array_equal(idx[c].cpu().numpy(), oracle.fps(cl, npoint))


def test_radius_counts(dev):
    """Padding rows hold copies of the key-points (they would fill the lowest bins).  ns > nt, ns == nt (the target is
    chosen) and ns == nt - 1, all inside one class: radii and m equal the exact call on the chosen cloud."""
    from bufferx_b200 import ops
    from bufferx_b200.synth import make_pair
    cap, Kr = 24576, 2000
    th = [5, 2, 0.5]
    d = make_pair("C2", 4, n_src=21000, n_tgt=21000)
    full = {0: d["src_fds_pcd"], 1: d["tgt_fds_pcd"]}
    for ns, nt in ((21000, 17000), (19000, 19000), (18000, 18001)):
        clouds = [full[0][:ns], full[1][:nt]]
        kps = [torch.from_numpy(c[np.random.default_rng(ns).choice(c.shape[0], Kr, replace=False)]).to(dev) for c in clouds]
        bufs = []
        for c, kp in zip(clouds, kps):
            b = kp.cpu().numpy()[np.arange(cap) % Kr].copy()             # poison: every padding row is a key-point
            b[:c.shape[0]] = c
            bufs.append(torch.from_numpy(b).to(dev))
        r, m, _ = ops.radius_estimate_pair(kps[0], bufs[0], kps[1], bufs[1], th, i32([ns, nt], dev))
        j = 0 if ns > nt else 1
        er, em, _ = ops.radius_estimate(kps[j], torch.from_numpy(np.ascontiguousarray(clouds[j])).to(dev), th)
        assert torch.equal(r, er) and torch.equal(m, em), (ns, nt, r, er)


@pytest.mark.parametrize("grid", [False, True])
def test_permute_and_select_patches_counts(dev, grid):
    """One launch, jobs of different N on both sides of GRID_MIN_POINTS inside the 16384 class, through the streaming scan
    and the hash grid.  Padding rows of the clouds hold the key-points (they would be the first hits); the permutation
    padding points at row 0.  Patches equal the exact calls bit for bit; rows beyond d_K and beyond the count stay
    untouched."""
    from bufferx_b200 import ops
    from bufferx_b200.synth import make_pair
    cap, K, P, k = 16384, 48, 64, 29
    sizes = [9000, 15000, 12000, 16384]
    assert min(sizes) < ops.GRID_MIN_POINTS <= max(sizes)
    rng = np.random.default_rng(9)
    exact, jobs, cnts = [], [], []
    for j, n in enumerate(sizes):
        pts = make_pair("C2", 10 + j, n_src=n)["src_fds_pcd"]
        kp = pts[rng.choice(n, K, replace=False)]
        perm = rng.permutation(n).astype(np.int32)
        buf = kp[np.arange(cap) % K].copy()
        buf[:n] = pts
        pbuf = np.zeros(cap, dtype=np.int32)
        pbuf[:n] = perm
        d_n = i32(n, dev)
        out4 = torch.full((cap, 4), NAN, device=dev)
        p4 = ops.permute_cloud(torch.from_numpy(buf).to(dev), torch.from_numpy(pbuf).to(dev), out4=out4, d_N=d_n)
        e4 = ops.permute_cloud(torch.from_numpy(pts).to(dev), torch.from_numpy(perm).to(dev))
        assert torch.equal(p4[:n], e4) and torch.isnan(p4[n:]).all()
        p4[n:] = torch.from_numpy(np.c_[kp[np.arange(cap - n) % K], np.zeros(cap - n, np.float32)]).to(dev)   # poison the permuted padding
        rad = torch.tensor([0.25 + 0.05 * j], device=dev)
        kpt = torch.from_numpy(kp).to(dev)
        jobs.append((p4, kpt, rad))
        exact.append((e4, kpt, rad))
        cnts.append(d_n)
    for c in (k, K):
        got = torch.full((len(sizes) * K, P, 3), NAN, device=dev)
        ops.select_patches_batched(jobs, P, got, grid=grid, d_K=[i32(c, dev)] * len(sizes), d_N=cnts)
        for j, (e4, kpt, rad) in enumerate(exact):
            ref = torch.empty((c, P, 3), device=dev)
            ops.select_patches_batched([(e4, kpt[:c].contiguous(), rad)], P, ref, grid=e4.shape[0] >= ops.GRID_MIN_POINTS)
            assert torch.equal(got[j * K:j * K + c], ref), (grid, sizes[j], c)
            assert torch.isnan(got[j * K + c:(j + 1) * K]).all()


# ------------------------------------------------------------------------------------------ model
def _cfg(name="C2", exit=False, iter_n=5000):
    from bufferx_b200.synth import workload_cfg
    cfg = workload_cfg(name)
    cfg.match.enable_early_exit = exit
    cfg.match.early_exit_min_inliers = 5
    cfg.match.iter_n = iter_n
    return cfg


@pytest.fixture(scope="module")
def state(dev):
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights
    return {k: v.detach().clone() for k, v in init_synthetic_weights(bx.BufferX(_cfg()), trained_pose=True).state_dict().items()}


def _model(cfg, sd, dev):
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights
    m = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True)
    if sd is not None:
        m.load_state_dict(sd)
    return m.to(dev).eval()


def _eq(a, b):
    return np.asarray(a[0]).tobytes() == np.asarray(b[0]).tobytes() and tuple(a[2:]) == tuple(b[2:])


def _run(model, items, in_flight):
    """items: [(data, perms)] -> [(result, slot)] with `in_flight` pairs launched ahead of the oldest result."""
    out, pending = [], []
    for d, p in items:
        if len(pending) == in_flight:
            h = pending.pop(0)
            out.append((h.result(), h))
        pending.append(model.forward_async(d, perms=p))
    out += [(h.result(), h) for h in pending]
    return out


def _shapes_served(items, results):
    served = {}
    for (d, _), (_, h) in zip(items, results):
        served.setdefault(id(h), set()).add((len(d["src_fds_pcd"]), len(d["tgt_fds_pcd"])))
    return served


def test_many_sizes_share_class_graphs(dev, oracle, state):
    """12 C2 pairs of distinct sizes (two classes, 9 k-point clouds on the hash grid of their class, the streaming scan
    eagerly), six in flight on class graphs: every result equals eager forward with the same perms."""
    from bufferx_b200 import ops
    from bufferx_b200.synth import make_pair
    cfg = _cfg()
    rng = np.random.default_rng(12)
    lo = rng.choice(np.arange(9000, 16384), size=(6, 2), replace=False)
    hi = rng.choice(np.arange(16385, 24000), size=(6, 2), replace=False)
    shapes = [tuple(int(v) for v in x) for pair in zip(lo, hi) for x in pair]       # alternating classes
    assert len(set(shapes)) == 12 and min(min(s) for s in shapes) < ops.GRID_MIN_POINTS
    items = [(make_pair("C2", 40 + i, n_src=a, n_tgt=b), oracle.draw_perms(cfg, a, b, 40 + i)) for i, (a, b) in enumerate(shapes)]
    model = _model(cfg, state, dev)
    with torch.no_grad():
        eager = [model(d, perms=p) for d, p in items]
        model.enable_cuda_graphs(True, slots_per_shape=3, size_classes=True)
        res = _run(model, items, 6)
        keys = {k: list(v) for k, v in model._slots.items()}
    model.enable_cuda_graphs(False)
    assert set(keys) == {(16384, 16384, False, False, None), (24576, 24576, False, False, None)}
    assert sum(len(v) for v in keys.values()) <= 2 * 3
    assert all(sl.graph is not None for v in keys.values() for sl in v)          # captured: no host sync in the path
    assert max(len(s) for s in _shapes_served(items, res).values()) >= 2
    for i, ((r, _), e) in enumerate(zip(res, eager)):
        assert _eq(r, e), (i, shapes[i], r[2:], e[2:])


def _unrelated(d, n):
    rng = np.random.default_rng(n)
    v = rng.normal(size=(n, 3))
    return dict(d, tgt_fds_pcd=(v / np.linalg.norm(v, axis=1, keepdims=True) * 0.7).astype(np.float32) + np.float32([0, 4, 1]))


def test_early_exit_pairs_share_a_class_graph(dev, oracle, state):
    """Exiting and non-exiting pairs of different sizes in the 24576 class, two in flight on one key: each result equals
    its exact-shape forward_async result."""
    from bufferx_b200.synth import make_pair
    cfg = _cfg(exit=True, iter_n=20000)
    shapes = [(20000, 20000), (17000, 23000), (22000, 18500), (19000, 21000), (24000, 16500), (18000, 18000)]
    items = []
    for i, (a, b) in enumerate(shapes):
        d = make_pair("C2", 3 + i, n_src=a, n_tgt=b)
        if i % 2:
            d = _unrelated(d, b)
        items.append((d, oracle.draw_perms(cfg, a, b, 3 + i)))
    model = _model(cfg, state, dev)
    with torch.no_grad():
        exact = [model.forward_async(d, perms=p).result() for d, p in items]
        model.enable_cuda_graphs(True, slots_per_shape=2, size_classes=True)
        res = _run(model, items, 2)
        keys = {k: list(v) for k, v in model._slots.items()}
    model.enable_cuda_graphs(False)
    assert list(keys) == [(24576, 24576, False, True, 5)] and len(keys[list(keys)[0]]) == 2
    assert {e[5] for e in exact} == {1, 3}
    for i, ((r, _), e) in enumerate(zip(res, exact)):
        assert _eq(r, e), (i, shapes[i], r[2:], e[2:])


def test_aligned_pairs_in_two_classes(dev, oracle, state):
    """C5-shaped z-aligned pairs: the source in the 65536 class, the target in the 32768 class."""
    from bufferx_b200.synth import make_pair
    cfg = _cfg("C5")
    items = []
    for i, (a, b) in enumerate([(60000, 30000), (57000, 31500)]):
        items.append((make_pair("C5", i, n_src=a, n_tgt=b), oracle.draw_perms(cfg, a, b, i)))
    model = _model(cfg, None, dev)
    with torch.no_grad():
        eager = [model(d, perms=p) for d, p in items]
        model.enable_cuda_graphs(True, slots_per_shape=1, size_classes=True)
        res = [model(d, perms=p) for d, p in items]        # forward() routes through the class slots
        keys = list(model._slots)
    model.enable_cuda_graphs(False)
    assert keys == [(65536, 32768, True, False, None)]
    for r, e in zip(res, eager):
        assert _eq(r, e), (r[2:], e[2:])


def _collate_dict(d):
    return {"src_fds_pcd": torch.from_numpy(d["src_fds_pcd"]), "tgt_fds_pcd": torch.from_numpy(d["tgt_fds_pcd"]),
            "relt_pose": torch.from_numpy(d["relt_pose"]), "src_id": d["src_id"], "tgt_id": d["tgt_id"], "scene_name": d["scene_name"],
            "sensor": d["sensor"], "voxel_sizes": torch.from_numpy(d["voxel_sizes"]), "dataset_names": list(d["dataset_names"]),
            "sphericity": torch.from_numpy(d["sphericity"]), "is_aligned_to_global_z": d["is_aligned_to_global_z"]}


def test_dataparallel_loop_with_size_classes(dev):
    """The drop-in loop of test_dropin (nn.DataParallel, NumPy's global RNG for the permutations, empty_cache between pairs,
    12 shapes): with size_classes=True every tuple equals eager's, and the 12 shapes run on one class graph."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, make_pair
    cfg = _cfg()
    cfg.patch.num_fps, cfg.patch.num_points_radius_estimate = 384, 512
    base = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True).to(dev)
    model = torch.nn.DataParallel(base, device_ids=[0])
    model.eval()
    rng = np.random.default_rng(7)
    shapes = [(int(rng.integers(4200, 6000)), int(rng.integers(4200, 6000))) for _ in range(12)]
    assert len(set(shapes)) == 12
    pairs = [make_pair("C1", 20 + i, n_src=a, n_tgt=b) for i, (a, b) in enumerate(shapes)]
    out = {}
    for classes in (None, True):
        base.enable_cuda_graphs(classes is not None, slots_per_shape=1, size_classes=bool(classes))
        out[classes] = []
        for i, d in enumerate(pairs):
            np.random.seed(100 + i)
            with torch.no_grad():
                out[classes].append(model(_collate_dict(d)))
            torch.cuda.empty_cache()
        if classes:
            assert list(base._slots) == [(8192, 8192, False, False, None)] and base._slots[(8192, 8192, False, False, None)][0].graph is not None
    base.enable_cuda_graphs(False)
    for i, (a, b) in enumerate(zip(out[True], out[None])):
        assert _eq(a, b), (i, shapes[i], a[2:], b[2:])


def test_inputs_from_another_stream_and_pinned(dev, oracle, state):
    """CUDA inputs produced on another stream and pinned host inputs, each into a class slot that a larger pair used
    before (its padding holds that pair's points)."""
    from bufferx_b200.synth import make_pair
    cfg = _cfg()
    model = _model(cfg, state, dev)
    big = make_pair("C2", 50, n_src=16000, n_tgt=16200)
    d = make_pair("C2", 51, n_src=10500, n_tgt=9800)
    perms_b, perms = oracle.draw_perms(cfg, 16000, 16200, 50), oracle.draw_perms(cfg, 10500, 9800, 51)
    with torch.no_grad():
        ref = model(d, perms=perms)
        model.enable_cuda_graphs(True, slots_per_shape=1, size_classes=True)
        src_h = torch.from_numpy(d["src_fds_pcd"]).pin_memory()
        tgt_h = torch.from_numpy(d["tgt_fds_pcd"]).pin_memory()
        burn = torch.empty(64 * 1024 * 1024, device=dev)
        side = torch.cuda.Stream(device=dev)
        outs = []
        for i in range(2):
            model.forward_async(big, perms=perms_b).result()
            with torch.cuda.stream(side):
                for _ in range(20):
                    burn.normal_()                                   # keep the producer stream busy before the H2D copies
                g = dict(d, src_fds_pcd=src_h.to(dev, non_blocking=True), tgt_fds_pcd=tgt_h.to(dev, non_blocking=True))
                outs.append(model.forward_async(g, perms=perms).result())
                del g
            model.forward_async(big, perms=perms_b).result()
            outs.append(model.forward_async(dict(d, src_fds_pcd=src_h, tgt_fds_pcd=tgt_h), perms=perms).result())
        assert list(model._slots) == [(16384, 16384, False, False, None)]
    model.enable_cuda_graphs(False)
    for o in outs:
        assert _eq(o, ref), (o[2:], ref[2:])


def test_fp16_fallback_in_a_class_slot(dev, oracle, state):
    """Point layer scaled so that features leave fp16 range: a class slot returns what eager forward returns after its own
    switch to the TF32 kernels, recomputed on the exact clouds."""
    from bufferx_b200.synth import make_pair
    sd = {k: v.clone() for k, v in state.items()}
    for k in ("pnt_layer.0.weight", "pnt_layer.0.bias", "pnt_layer.1.running_mean", "pnt_layer.1.bias"):
        sd["Desc." + k] = sd["Desc." + k] * 1.0e6
    cfg = _cfg()
    d = make_pair("C2", 52, n_src=17500, n_tgt=21000)
    perms = oracle.draw_perms(cfg, 17500, 21000, 52)
    with torch.no_grad():
        m1 = _model(cfg, sd, dev)
        m1.enable_cuda_graphs(True, slots_per_shape=1, size_classes=True)
        got = m1.forward_async(d, perms=perms).result()
        assert m1.Desc.conv_net.force_tf32
        m1.enable_cuda_graphs(False)
        m2 = _model(cfg, sd, dev)
        exp = m2(d, perms=perms)
        assert m2.Desc.conv_net.force_tf32
    assert _eq(got, exp)
