"""FPS of clouds beyond one cluster's registers (bx_fps_large, N > 524288) and the pairs that need it.

ops.fps_large must equal the C oracle bit for bit (indices, and key points = xyz[idx]) on synthetic clouds up to the
1638400-point limit, on the edge clouds of oracle/frontend_cases.py (also held to float64), and on small clouds, where it
must also equal ops.fps.  Whole pairs with one or both clouds above 524288 points go through BufferX.forward against the
oracle pair, and through captured slots, exact-shape and size-class, against eager forward.

Both clouds of such a pair exceed 200000 points, so each scale's radius estimation histograms 200000 indices the reference
draws with torch.randint (BUFFERX.py:664-665), one draw per scale.  The tests pin those draws to fixed sets per cloud size,
a distinct one per scale -- in eager forward, in the captures (which otherwise draw on the device, DESIGN.md section 2) and
in the oracle -- so that every route sees the same sub-samples and results can be compared byte for byte."""
import functools
import os
import sys

import numpy as np
import pytest
import torch

from oracle import frontend_cases as F

pytestmark = pytest.mark.gpu
LIMIT = 1638400


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


def cu(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)


def _same_as_oracle(oracle, x, npoint):
    from bufferx_b200 import ops
    idx, kp = ops.fps_large(x, npoint)
    want = oracle.fps(x.cpu().numpy(), npoint)
    got = idx.cpu().numpy()
    assert np.array_equal(got, want), f"first difference at step {int(np.flatnonzero(got != want)[0])}"
    assert torch.equal(kp, x[idx.long()]), "kpts != xyz[idx]"
    return idx, kp


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("n", [524289, 1048576, LIMIT])
def test_fps_large_synthetic_clouds(dev, oracle, n):
    from bufferx_b200.synth import make_pair
    x = cu(make_pair("C3", 7, n_src=n, n_tgt=1000)["src_fds_pcd"], dev)
    _same_as_oracle(oracle, x, 2000)


@pytest.mark.parametrize("kind", ["equal", "lattice", "dup", "allskip", "fewvalid", "magedge", "offset"])
def test_fps_large_edge_clouds(dev, oracle, kind):
    """600000 points: all equal (the tie rule alone decides), lattice and duplicate ties, every point or all but a few
    inside the 1e-3 skip, magnitudes either side of it, and a cloud 1e4 m from the origin."""
    n = 600000
    if kind == "equal":
        xyz = np.tile(np.float32([[1.5, -0.25, 0.75]]), (n, 1))
    elif kind == "offset":
        xyz = F.fps_cloud("uniform", n, seed=3, offset=1e4)
    else:
        xyz = F.fps_cloud(kind, n, seed=3, k_valid=50)
    x = cu(xyz, dev)
    idx, kp = _same_as_oracle(oracle, x, 2000)
    F.report(f"fps_large {kind}", F.check_fps(x, 2000, idx, kp))


@pytest.mark.parametrize("n", [1, 4097, 524288])
def test_fps_large_equals_fps_where_both_run(dev, oracle, n):
    from bufferx_b200 import ops
    x = cu(F.fps_cloud("dup" if n > 1 else "uniform", n, seed=n), dev)
    npoint = 5 if n == 1 else 2000
    idx, kp = _same_as_oracle(oracle, x, npoint)
    ref, ref_kp = ops.fps(x, [0, n], npoint)
    assert torch.equal(idx, ref[0]) and torch.equal(kp, ref_kp[0])


def test_fps_large_refuses_beyond_the_limit(dev):
    from bufferx_b200 import ops
    x = torch.zeros((LIMIT + 1, 3), dtype=torch.float32, device=dev)
    before = ops.launch_count()
    with pytest.raises(ops.BufferXError, match="1638400"):
        ops.fps_large(x, 16)
    assert ops.launch_count() == before


# ------------------------------------------------------------------------------------------------ pairs
def _cfg():
    from bufferx_b200.synth import workload_cfg
    cfg = workload_cfg("C3")
    cfg.patch.num_fps, cfg.patch.num_points_radius_estimate, cfg.match.iter_n = 300, 600, 5000
    cfg.match.enable_early_exit = False
    return cfg


_SUBS = {}
SCALES = 3      # the C3 configuration's scales: a pair draws one sub-sample per scale


def _sub(n, k=0, device="cpu"):
    """The k-th fixed 200000-index sub-sample of an n-point cloud, k < SCALES, all distinct (so that scales sharing one
    draw would be seen); device copies are made outside any capture and kept."""
    key = (n, k, str(torch.device(device)))
    if key not in _SUBS:
        assert torch.device(device).type == "cpu" or not torch.cuda.is_current_stream_capturing()
        _SUBS[key] = torch.from_numpy(np.random.default_rng([n, k]).integers(0, n, 200000)).to(device)
    return _SUBS[key]


@pytest.fixture
def pinned_draw(monkeypatch):
    """torch.randint(0, n, (200000,)) returns the pinned draws of an n-point cloud in turn (0, 1, .., SCALES - 1, 0, ..),
    so every pair -- eager forward, a capture, a slot launch, the oracle's per-scale draws -- takes draw i at scale i."""
    randint = torch.randint
    turn = {}

    def fixed(*a, **kw):
        if len(a) >= 3 and a[0] == 0 and tuple(a[2]) == (200000,):
            n, device = int(a[1]), kw.get("device", "cpu")
            k = turn.get(n, 0)
            turn[n] = (k + 1) % SCALES
            return _sub(n, k, device)
        return randint(*a, **kw)

    monkeypatch.setattr(torch, "randint", fixed)


PAIRS = [(700000, 600000), (560000, 300000)]


@functools.lru_cache(maxsize=None)
def _pair(ns, nt):
    from bufferx_b200.synth import make_pair
    return make_pair("C3", 11, n_src=ns, n_tgt=nt)


def _model(dev):
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights
    model = init_synthetic_weights(bx.BufferX(_cfg()), seed=7)
    return model, {k: v.detach().clone() for k, v in model.state_dict().items()}


@pytest.mark.parametrize("ns,nt", PAIRS)
def test_large_pair_against_the_oracle(dev, oracle, pinned_draw, monkeypatch, ns, nt):
    """Key points, radii, neighbour lists, voxel selections and LRFs equal; descriptors, matches and the pose within the
    bars of the whole-pair tests (tests/test_gpu_parity.py)."""
    from bufferx_b200 import ops
    here = os.path.dirname(os.path.abspath(__file__))
    if here not in sys.path:
        sys.path.insert(0, here)
    from test_gpu_parity import _compare_pair
    calls = []
    fps_large = ops.fps_large

    def rec(xyz, *a, **kw):
        calls.append(xyz.shape[0])
        return fps_large(xyz, *a, **kw)

    model, sd = _model(dev)
    cfg, data = model.config, _pair(ns, nt)
    perms = oracle.draw_perms(cfg, ns, nt, 0)
    monkeypatch.setattr(ops, "fps_large", rec)
    _compare_pair(model.to(dev), sd, cfg, data, perms, oracle, f"C3 {ns}/{nt}")
    monkeypatch.setattr(ops, "fps_large", fps_large)
    assert calls == [n for n in (ns, nt) if n > ops.FPS_MAX_POINTS]
    model.cpu()


def _eq(a, b):
    return np.asarray(a[0]).tobytes() == np.asarray(b[0]).tobytes() and tuple(a[2:]) == tuple(b[2:])


@pytest.mark.parametrize("size_classes", [False, True])
def test_large_pairs_on_captured_slots(dev, oracle, pinned_draw, size_classes):
    """Each pair through enable_cuda_graphs(True) + forward_async, its graph replayed twice, and through forward on the
    same slots: the bytes of eager forward."""
    model, _ = _model(dev)
    model = model.to(dev).eval()
    items = [(_pair(ns, nt), oracle.draw_perms(model.config, ns, nt, 1)) for ns, nt in PAIRS]
    for ns, nt in PAIRS:
        for k in range(SCALES):
            _sub(max(ns, nt), k, dev)   # the device copies the captures index with, made before any capture
    with torch.no_grad():
        eager = [model(d, perms=p) for d, p in items]
        model.enable_cuda_graphs(True, slots_per_shape=1, size_classes=size_classes)
        try:
            for (d, p), e in zip(items, eager):
                for _ in range(2):
                    assert _eq(model.forward_async(d, perms=p).result(), e)
                assert _eq(model(d, perms=p), e)
            slots = [sl for v in model._slots.values() for sl in v]
            assert len(slots) == len(PAIRS) and all(sl.graph is not None and not sl.counted for sl in slots)
        finally:
            model.enable_cuda_graphs(False)
    model.cpu()


def test_forward_refuses_beyond_the_limit(dev):
    """A 1638401-point cloud: BufferXError naming the limit from forward and forward_async, before any launch."""
    from bufferx_b200 import ops
    model, _ = _model(dev)
    model = model.to(dev).eval()
    rng = np.random.default_rng(0)
    small = rng.uniform(-5, 5, (1000, 3)).astype(np.float32)
    big = rng.uniform(-5, 5, (LIMIT + 1, 3)).astype(np.float32)
    before = ops.launch_count()
    for src, tgt in ((big, small), (small, big)):
        data = dict(src_fds_pcd=src, tgt_fds_pcd=tgt, is_aligned_to_global_z=True)
        with torch.no_grad():
            with pytest.raises(ops.BufferXError, match="1638400"):
                model(data)
            with pytest.raises(ops.BufferXError, match="1638400"):
                model.forward_async(data)
    torch.cuda.synchronize()
    assert ops.launch_count() == before
    model.cpu()
