"""Size-class slots for pairs with clouds above 200000 points (enable_cuda_graphs(True, size_classes=True,
large_classes=True)) and the two device forms they run on.

  * ops.fps_large with a device count (bx_fps_large_n) on a capacity buffer whose padding rows would win if they were read:
    the indices and key-points of ops.fps_large on the exact cloud, also when one captured launch is replayed with two counts.
  * ops.radius_estimate_pair with the 200000-index sub-sample (bx_radius_estimate_n_sub): the histogram, radii and m of
    ops.radius_estimate on the gathered larger cloud with denom = N * Kr; with one sub-sample per scale ([S, 200000], one
    launch per scale) each scale's histogram, radius and m on its own gathered cloud.
  * Whole pairs through large-class slots: with the same perms and the same torch.manual_seed, the bytes of eager forward.
    The sub-samples are the reference's own torch.randint draws on the CPU generator, one per scale, made by eager
    forward and by each slot launch alike; nothing is pinned here."""
import functools

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
LIMIT = 1638400
SUB = 200000


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


@functools.lru_cache(maxsize=None)
def _cloud(n, seed=7):
    from bufferx_b200.synth import make_pair
    return make_pair("C3", seed, n_src=n, n_tgt=1000)["src_fds_pcd"]


def _poisoned(x, cap, dev, poison):
    """x [n,3] in the first rows of a [cap,3] CUDA buffer; the padding rows cycle through `poison` ([k,3])."""
    buf = torch.empty((cap, 3), dtype=torch.float32)
    n = x.shape[0]
    buf[:n] = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
    if cap > n:
        p = torch.as_tensor(poison, dtype=torch.float32).reshape(-1, 3)
        buf[n:] = p[torch.arange(cap - n) % p.shape[0]]
    return buf.to(dev)


FPS_POISON = [[float("nan")] * 3, [1e6, 1e6, 1e6], [-1e6, 3e5, 1e6], [float("nan"), 0.0, 0.0]]


# ------------------------------------------------------------------------------------------------ FPS count form
@pytest.mark.parametrize("n,cap", [(1, 645120), (524289, 645120), (600001, 645120), (1048576, 1216512), (LIMIT, LIMIT)])
def test_fps_count_form(dev, n, cap):
    from bufferx_b200 import ops
    buf = _poisoned(_cloud(max(n, 1000))[:n], cap, dev, FPS_POISON)
    d_n = torch.tensor([n], dtype=torch.int32, device=dev)
    idx, kp = ops.fps_large(buf, 2000, d_count=d_n)
    ref, ref_kp = ops.fps_large(buf[:n].contiguous(), 2000)
    assert torch.equal(idx, ref), f"first difference at step {int((idx != ref).nonzero()[0])}"
    assert torch.equal(kp.view(torch.int32), ref_kp.view(torch.int32))


def test_fps_count_form_graph_replayed_with_two_counts(dev):
    """One captured launch on a 792576-point capacity, replayed on a 780000-point cloud, a 645121-point cloud and the
    first again, each time with the padding poisoned."""
    from bufferx_b200 import ops
    cap = 792576
    clouds = [_poisoned(_cloud(n, seed)[:n], cap, dev, FPS_POISON) for n, seed in ((780000, 5), (645121, 6))]
    refs = [ops.fps_large(c[:n].contiguous(), 2000) for c, n in zip(clouds, (780000, 645121))]
    buf = clouds[0].clone()
    d_n = torch.tensor([780000], dtype=torch.int32, device=dev)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        ops.fps_large(buf, 2000, d_count=d_n)             # warm-up: kernel attributes are set outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = ops.fps_large(buf, 2000, d_count=d_n)
    for k, n in ((0, 780000), (1, 645121), (0, 780000)):
        buf.copy_(clouds[k])
        d_n.fill_(n)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out[0], refs[k][0]), n
        assert torch.equal(out[1].view(torch.int32), refs[k][1].view(torch.int32)), n


# ------------------------------------------------------------------------------------------------ radius, sub-sampled
RADIUS_CASES = [
    ((700000, 300000), (792576, 524288)),     # source chosen
    ((250000, 900000), (262144, 976896)),     # target chosen
    ((600000, 600000), (645120, 645120)),     # ns == nt: the target
    ((200000, 5000), (262144, 8192)),         # at the sub-sample limit: the whole cloud, d_sub not read
    ((200001, 5000), (262144, 8192)),         # one above it, in the same capacity
]


@pytest.mark.parametrize("counts,caps", RADIUS_CASES)
def test_radius_sub_sampled_pair_form(dev, counts, caps):
    from bufferx_b200 import ops
    from bufferx_b200.synth import workload_cfg
    thresholds = workload_cfg("C3").patch.search_radius_thresholds
    Kr = 2000
    (ns, nt), (cs, ct) = counts, caps
    g = torch.Generator().manual_seed(ns + nt)
    clouds, kpts = [], []
    for n, cap, seed in ((ns, cs, 3), (nt, ct, 4)):
        x = _cloud(n, seed)[:n]
        k = torch.from_numpy(x[torch.randint(0, n, (Kr,), generator=g).numpy()]).to(dev).contiguous()
        clouds.append(_poisoned(x, cap, dev, k.cpu()))     # padding rows on the key-points: each would count if read
        kpts.append(k)
    N = ns if ns > nt else nt
    pts_r, kpts_r = (clouds[0], kpts[0]) if ns > nt else (clouds[1], kpts[1])
    sub = torch.randint(0, N, (SUB,), generator=g)
    d_sub = sub.to(dev, torch.int32)
    if ns == 200000:
        d_sub.fill_(-1)       # not read: any value would do
    d_counts = torch.tensor([ns, nt], dtype=torch.int32, device=dev)
    r, m, hist = ops.radius_estimate_pair(kpts[0], clouds[0], kpts[1], clouds[1], thresholds, d_counts, d_sub=d_sub)
    pts_e = pts_r[:N][sub.to(dev)].contiguous() if N > SUB else pts_r[:N].contiguous()
    r_e, m_e, hist_e = ops.radius_estimate(kpts_r, pts_e, thresholds, denom=N * Kr)
    assert torch.equal(hist, hist_e)
    assert torch.equal(m, m_e) and torch.equal(r.view(torch.int32), r_e.view(torch.int32))
    assert int(hist_e[-2]) > 0


@pytest.mark.parametrize("counts,caps", RADIUS_CASES)
def test_radius_sub_sampled_pair_form_per_scale(dev, counts, caps):
    """d_sub [S, 200000], one sub-sample per scale: scale i's histogram, radius and m are those of ops.radius_estimate on
    its own gathered cloud with its own threshold (the padding rows of both buffers would count if read)."""
    from bufferx_b200 import ops
    from bufferx_b200.synth import workload_cfg
    thresholds = workload_cfg("C3").patch.search_radius_thresholds
    S = len(thresholds)
    Kr = 2000
    (ns, nt), (cs, ct) = counts, caps
    g = torch.Generator().manual_seed(ns + nt)
    clouds, kpts = [], []
    for n, cap, seed in ((ns, cs, 3), (nt, ct, 4)):
        x = _cloud(n, seed)[:n]
        k = torch.from_numpy(x[torch.randint(0, n, (Kr,), generator=g).numpy()]).to(dev).contiguous()
        clouds.append(_poisoned(x, cap, dev, k.cpu()))     # padding rows on the key-points: each would count if read
        kpts.append(k)
    N = ns if ns > nt else nt
    pts_r, kpts_r = (clouds[0], kpts[0]) if ns > nt else (clouds[1], kpts[1])
    sub = torch.randint(0, N, (S, SUB), generator=g)
    d_sub = sub.to(dev, torch.int32)
    if ns == 200000:
        d_sub.fill_(-1)       # not read: any value would do
    d_counts = torch.tensor([ns, nt], dtype=torch.int32, device=dev)
    r, m, hist = ops.radius_estimate_pair(kpts[0], clouds[0], kpts[1], clouds[1], thresholds, d_counts, d_sub=d_sub)
    assert tuple(hist.shape) == (S, ops.RADIUS_BINS + 2)
    for i in range(S):
        pts_e = pts_r[:N][sub[i].to(dev)].contiguous() if N > SUB else pts_r[:N].contiguous()
        r_e, m_e, hist_e = ops.radius_estimate(kpts_r, pts_e, thresholds[i:i + 1], denom=N * Kr)
        assert torch.equal(hist[i], hist_e), f"scale {i}: histogram"
        assert torch.equal(m[i:i + 1], m_e) and torch.equal(r[i:i + 1].view(torch.int32), r_e.view(torch.int32)), f"scale {i}: radius"
        assert int(hist_e[-2]) > 0
    if N > SUB:     # three draws, three histograms
        assert not torch.equal(hist[0], hist[1]) and not torch.equal(hist[1], hist[2])
    with pytest.raises(ops.BufferXError, match="d_sub must be"):
        ops.radius_estimate_pair(kpts[0], clouds[0], kpts[1], clouds[1], thresholds, d_counts, d_sub=d_sub[:2])


# ------------------------------------------------------------------------------------------------ whole pairs
def _cfg(early_exit=False):
    from bufferx_b200.synth import workload_cfg
    cfg = workload_cfg("C3")
    cfg.patch.num_fps, cfg.patch.num_points_radius_estimate, cfg.match.iter_n = 300, 600, 5000
    cfg.match.enable_early_exit = early_exit
    return cfg


# distinct sizes between 200001 and 1638400 points; the first two share a class key
PAIRS = [(700000, 600000), (760000, 640000), (LIMIT, 250000), (300000, 1000000), (210000, 20000), (550000, 540000)]


@functools.lru_cache(maxsize=None)
def _pair(ns, nt):
    from bufferx_b200.synth import make_pair
    return make_pair("C3", 11, n_src=ns, n_tgt=nt)


def _model(dev, early_exit=False):
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights
    return init_synthetic_weights(bx.BufferX(_cfg(early_exit)), seed=7).to(dev).eval()


def _eq(a, b):
    return np.asarray(a[0]).tobytes() == np.asarray(b[0]).tobytes() and tuple(a[2:]) == tuple(b[2:])


def _seeded(seed, fn, *a, **kw):
    torch.manual_seed(seed)
    return fn(*a, **kw)


def test_large_pairs_on_class_slots(dev, oracle):
    model = _model(dev)
    items = [(_pair(ns, nt), oracle.draw_perms(model.config, ns, nt, 1)) for ns, nt in PAIRS]
    with torch.no_grad():
        eager = [_seeded(100 + i, model, d, perms=p) for i, (d, p) in enumerate(items)]
        model.enable_cuda_graphs(True, slots_per_shape=1, size_classes=True, large_classes=True)
        try:
            for i, ((d, p), e) in enumerate(zip(items, eager)):
                for _ in range(2):
                    assert _eq(_seeded(100 + i, lambda: model.forward_async(d, perms=p).result()), e), PAIRS[i]
                assert _eq(_seeded(100 + i, model, d, perms=p), e), PAIRS[i]
            slots = [sl for v in model._slots.values() for sl in v]
            assert len(slots) < len(PAIRS)
            assert all(sl.graph is not None and sl.counted and sl.sub is not None for sl in slots)
        finally:
            model.enable_cuda_graphs(False)
    model.cpu()


def test_large_pairs_with_early_exit(dev, oracle):
    """Early exit decided on the device: graph and no-graph large-class slots give the same bytes."""
    model = _model(dev, early_exit=True)
    pairs = PAIRS[:3]
    items = [(_pair(ns, nt), oracle.draw_perms(model.config, ns, nt, 2)) for ns, nt in pairs]
    out = {}
    with torch.no_grad():
        for graphs in (False, True):
            model.enable_cuda_graphs(graphs, slots_per_shape=1, size_classes=True, large_classes=True)
            try:
                out[graphs] = [_seeded(200 + i, lambda: model.forward_async(d, perms=p).result()) for i, (d, p) in enumerate(items)]
                slots = [sl for v in model._slots.values() for sl in v]
                assert len(slots) < len(pairs) and all(sl.counted and (sl.graph is not None) == graphs for sl in slots)
            finally:
                model.enable_cuda_graphs(False)
    for a, b, pr in zip(out[False], out[True], pairs):
        assert _eq(a, b), pr
    model.cpu()


def test_large_classes_refuse_beyond_the_limit(dev):
    """A 1638401-point cloud: BufferXError naming the limit from forward and forward_async, before any launch."""
    from bufferx_b200 import ops
    model = _model(dev)
    model.enable_cuda_graphs(True, size_classes=True, large_classes=True)
    rng = np.random.default_rng(0)
    small = rng.uniform(-5, 5, (1000, 3)).astype(np.float32)
    big = rng.uniform(-5, 5, (LIMIT + 1, 3)).astype(np.float32)
    torch.cuda.synchronize()
    before = ops.launch_count()
    for src, tgt in ((big, small), (small, big)):
        data = dict(src_fds_pcd=src, tgt_fds_pcd=tgt, is_aligned_to_global_z=True)
        with torch.no_grad():
            with pytest.raises(ops.BufferXError, match="1638400"):
                model(data)
            with pytest.raises(ops.BufferXError, match="1638400"):
                model.forward_async(data)
    torch.cuda.synchronize()
    assert ops.launch_count() == before and not model._slots
    model.enable_cuda_graphs(False)
    model.cpu()
