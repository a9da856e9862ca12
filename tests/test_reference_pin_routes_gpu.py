"""The CUDA path against the reference's own ``BufferX.forward`` on the routes beside C2 (tests/golden/<route>_seed<k>_
reference.npz, written by oracle/ref_check.py; see tests/test_reference_pin_routes_cpu.py): the outdoor route (C3, C5),
clouds above 200000 points (C3L, C3LT, C3LE) and early exit (C2E, C2N).

Eager ``forward`` after torch.manual_seed(seed): FPS indices and per-scale radii equal, >= 99.5 % of the reference's mutual
matches, the consensus set equal, counts equal (|d num_mutual| <= 2), RANSAC T within 1e-6, pose within 0.1 deg / 5 mm, and
torch's CPU generator left where the reference left it.  Above 200000 points the same pair through large-class slots
(forward_async) equals the reference too; early-exit pairs through forward_async (decided on the device) agree in scales
used, counts and pose."""
import functools
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
FIXTURES = [("C3", 0), ("C3", 1), ("C5", 0), ("C3L", 0), ("C3LT", 0), ("C3LE", 0), ("C2E", 0), ("C2N", 0)]
LARGE = [f for f in FIXTURES if f[0].startswith("C3L")]
EXITS = [f for f in FIXTURES if f[0] in ("C2E", "C2N", "C3LE")]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


def _ref(name, seed):
    return np.load(os.path.join(GOLD, f"{name.lower()}_seed{seed}_reference.npz"))


@functools.lru_cache(maxsize=None)
def _setup(name, seed):
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights
    from oracle import oracle as O
    from oracle.ref_check import route_cfg, route_pair
    r = _ref(name, seed)
    cfg = route_cfg(name)
    if cfg.match.enable_early_exit:
        cfg.match.early_exit_min_inliers = int(r["early_exit_min_inliers"])
    data = route_pair(name, seed)
    perms = O.draw_perms(cfg, int(r["n_src"]), int(r["n_tgt"]), seed)
    return cfg, data, perms, init_synthetic_weights(bx.BufferX(cfg), trained_pose=True).state_dict()


def _model(name, seed, dev):
    import bufferx_b200 as bx
    cfg, data, perms, sd = _setup(name, seed)
    model = bx.BufferX(cfg)
    model.load_state_dict(sd)
    return model.to(dev).eval(), data, perms


def _rng_sha():
    from oracle.ref_check import sha
    return sha(torch.get_rng_state().numpy())


def _check_result(r, out):
    from bufferx_b200.se3 import compute_rre, compute_rte
    pose, _, ninl, nmut, nind, su = out
    assert [ninl, nind, su] == [int(r["counts"][0]), int(r["counts"][2]), int(r["counts"][3])]
    assert abs(nmut - int(r["counts"][1])) <= 2
    assert compute_rre(pose, r["pose"]) < 0.1 and compute_rte(pose, r["pose"]) < 0.005


@pytest.mark.parametrize("name,seed", FIXTURES)
def test_forward_against_the_reference_forward_on_route(dev, name, seed):
    r = _ref(name, seed)
    model, data, perms = _model(name, seed, dev)
    torch.manual_seed(seed)
    with torch.no_grad():
        out = model(data, perms=perms, ransac_seed=0, debug=True)
    assert _rng_sha() == bytes(r["rng_state_sha"]).decode(), "torch's generator is not where the reference leaves it"
    dbg = model.last_debug
    assert (dbg["fps_idx"][0].cpu().numpy() == r["s_fps"]).all() and (dbg["fps_idx"][1].cpu().numpy() == r["t_fps"]).all()
    su = out[5]
    des_r = dbg["des_r"].cpu().numpy()[:su]           # float32: the reference's 2-decimal radius, rounded once
    assert des_r.tolist() == r["des_r"].astype(np.float32).tolist(), f"radii {des_r.tolist()} != {r['des_r'].tolist()}"
    common = total = 0
    for i, sc in enumerate(dbg["scales"]):
        M = int(sc["dM"].item())
        gs = set(zip(sc["s_mids"][:M].cpu().numpy().tolist(), sc["t_mids"][:M].cpu().numpy().tolist()))
        rs = set(zip(r[f"s{i}_s_mids"].tolist(), r[f"s{i}_t_mids"].tolist()))
        common += len(gs & rs)
        total += len(rs)
    assert common >= 0.995 * total
    last = dbg["scales"][-1]
    inl = last["inlier_ind"][:int(last["dI"].item())].cpu().numpy()
    assert np.array_equal(inl, r["inlier_ind"]), "consensus set differs from the reference run's"
    assert np.abs(np.asarray(dbg["init_pose"]) - r["ransac_T"]).max() < 1e-6
    _check_result(r, out)
    assert np.abs(r["pose"] - np.eye(4)).max() > 1e-3                    # non-vacuous


@pytest.mark.parametrize("name,seed", LARGE)
def test_large_class_slots_against_the_reference_forward(dev, name, seed):
    """enable_cuda_graphs(True, size_classes=True, large_classes=True) + forward_async after torch.manual_seed(seed): the
    launch draws the S sub-samples the reference draws (scale i on draw i), so the replayed pair equals the reference,
    and eager forward byte for byte."""
    r = _ref(name, seed)
    model, data, perms = _model(name, seed, dev)
    with torch.no_grad():
        torch.manual_seed(seed)
        eager = model(data, perms=perms)
        model.enable_cuda_graphs(True, slots_per_shape=1, size_classes=True, large_classes=True)
        try:
            for _ in range(2):                  # the capture, then a replay
                torch.manual_seed(seed)
                out = model.forward_async(data, perms=perms).result()
                _check_result(r, out)
                assert np.array_equal(np.asarray(out[0]), np.asarray(eager[0])) and out[2:] == eager[2:]
                if int(r["counts"][3]) == 3:    # without an exit the launch's S draws are the reference's
                    assert _rng_sha() == bytes(r["rng_state_sha"]).decode()
            assert all(sl.sub is not None for v in model._slots.values() for sl in v)
        finally:
            model.enable_cuda_graphs(False)


@pytest.mark.parametrize("name,seed", EXITS)
def test_forward_async_early_exit_against_the_reference_forward(dev, name, seed):
    """The exit decided on the device (forward_async, captured): the reference's scales used, counts and pose."""
    r = _ref(name, seed)
    model, data, perms = _model(name, seed, dev)
    large = name.startswith("C3L")
    with torch.no_grad():
        model.enable_cuda_graphs(True, slots_per_shape=1, size_classes=large, large_classes=large)
        try:
            for _ in range(2):
                torch.manual_seed(seed)
                _check_result(r, model.forward_async(data, perms=perms).result())
        finally:
            model.enable_cuda_graphs(False)
