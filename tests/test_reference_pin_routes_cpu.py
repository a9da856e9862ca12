"""The oracle against the reference's own ``BufferX.forward`` on the routes beside C2: the outdoor route (C3 / KITTI, C5 /
TIERS_hetero: aligned, confidence 1.0, no refinement), clouds above 200000 points (C3L, C3LT, C3LE), and early exit
(C2E exits at scale 0, C2N does not).  tests/golden/<route>_seed<k>_reference.npz were written by oracle/ref_check.py from
the reference's forward (the outdoor routes in a reduced variant: 300 key-points, 600 radius key-points, 5000 RANSAC
iterations, the cloud sizes and the 200000-point cut as configured; C2E / C2N in the full C2 configuration).  Every discrete result must be equal: FPS indices, per-scale radii, match lists,
every RANSAC call's consensus set, count and T, scales used, counts and pose, and above 200000 points the radius
sub-samples drawn from torch's CPU generator (count, sha of each draw, sha of the generator state afterwards).

Each test below the replay applies one plausible mistake to the oracle and shows that the same check rejects it."""
import functools
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
FIXTURES = [("C3", 0), ("C3", 1), ("C5", 0), ("C3L", 0), ("C3LT", 0), ("C3LE", 0), ("C2E", 0), ("C2N", 0)]


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
    sd = {k: v.detach().clone() for k, v in init_synthetic_weights(bx.BufferX(cfg), trained_pose=True).state_dict().items()}
    data = route_pair(name, seed)
    assert (len(data["src_fds_pcd"]), len(data["tgt_fds_pcd"])) == (int(r["n_src"]), int(r["n_tgt"]))
    perms = O.draw_perms(cfg, int(r["n_src"]), int(r["n_tgt"]), seed)
    return cfg, sd, data, perms


def _replay(oracle, name, seed):
    """The oracle as ref_check.py ran the reference: torch.manual_seed(seed) before the pair, the reference's LRF z axes
    imposed off the aligned route (its covariance is a BLAS sum whose order is not in its source)."""
    from oracle.ref_check import RandintLog, sha
    cfg, sd, data, perms = _setup(name, seed)
    r = _ref(name, seed)
    S = cfg.patch.num_scales
    z_axes = None
    if "s0_src_z" in r:
        z_axes = [(r[f"s{i}_src_z"], r[f"s{i}_tgt_z"]) if f"s{i}_src_z" in r else (None, None) for i in range(S)]
    hist, clouds = oracle.radius_hist, []

    def rec_hist(kpts, pts):          # which key-points and points each radius histogram measured
        clouds.append(sha(np.ascontiguousarray(kpts, np.float32)) + sha(np.ascontiguousarray(pts, np.float32)))
        return hist(kpts, pts)

    oracle.radius_hist = rec_hist
    torch.manual_seed(seed)
    try:
        with RandintLog() as draws:
            out = oracle.register_pair(sd, cfg, data, perms, 0, keep=True, z_axes=z_axes)
    finally:
        oracle.radius_hist = hist
    draws.clouds = clouds
    return out, draws


@functools.lru_cache(maxsize=None)
def _clean_replay(name, seed):
    from oracle import oracle as O
    O.build()
    return _replay(O, name, seed)


def _check(name, seed, out, draws):
    r = _ref(name, seed)
    pose, ninl, nmut, nind, su, aux = out
    assert (aux["s_fps"] == r["s_fps"]).all() and (aux["t_fps"] == r["t_fps"]).all(), "FPS indices"
    assert su == int(r["counts"][3]), f"scales used {su} != {int(r['counts'][3])}"
    assert aux["des_r"][:su] == r["des_r"].tolist(), f"radii {aux['des_r']} != {r['des_r'].tolist()}"
    for i in range(su):
        sc = aux["scales"][i]
        assert np.array_equal(sc["s_mids"], r[f"s{i}_s_mids"]) and np.array_equal(sc["t_mids"], r[f"s{i}_t_mids"]), f"scale {i} matches"
    calls = aux["ransac_calls"]
    assert len(calls) == int(r["n_ransac"]), "number of RANSAC calls"
    for k, c in enumerate(calls):
        assert np.array_equal(c["inlier_ind"], r[f"ransac{k}_inlier_ind"]), f"RANSAC call {k}: consensus set"
        assert c["num_inliers"] == int(r[f"ransac{k}_num_inliers"]), f"RANSAC call {k}: inliers"
        assert np.abs(c["T"] - r[f"ransac{k}_T"]).max() <= 1e-12, f"RANSAC call {k}: T"
    assert [ninl, nmut, nind, su] == r["counts"].tolist()
    if _setup(name, seed)[0].test.pose_refine:
        # the reference refines in torch, the oracle restates it in C: the same rounds, sums in another order
        assert np.abs(np.asarray(pose, np.float64) - r["pose"]).max() < 1e-5, "refined pose"
    else:
        assert np.array_equal(np.asarray(pose, np.float64), r["pose"]), "pose"
    assert len(draws.shas) == int(r["n_draws"]), f"{len(draws.shas)} sub-sample draws, the reference made {int(r['n_draws'])}"
    assert draws.shas == [bytes(r[f"draw{k}_sha"]).decode() for k in range(int(r["n_draws"]))], "sub-sample draws"
    assert draws.state_sha == bytes(r["rng_state_sha"]).decode(), "torch generator state after the pair"
    if int(r["n_draws"]):           # above 200000 points: one histogram per scale, over the reference's cloud and sample
        assert draws.clouds == [bytes(r[f"radius{k}_cloud_sha"]).decode() for k in range(su)], "radius key-points / points"


@pytest.mark.parametrize("name,seed", FIXTURES)
def test_oracle_equals_reference_forward_on_route(name, seed):
    r = _ref(name, seed)
    out, draws = _clean_replay(name, seed)
    _check(name, seed, out, draws)
    # what makes each pin non-vacuous
    assert np.abs(r["pose"] - np.eye(4)).max() > 1e-3, "the reference's pose is the identity"
    if name in ("C3L", "C3LT"):
        assert int(r["n_draws"]) == 3
    if name in ("C3LE", "C2E"):
        assert int(r["counts"][3]) == 1 and int(r["n_ransac"]) == 1
        assert int(r["ransac0_num_inliers"]) == int(r["early_exit_min_inliers"]), "the exit is on the >= boundary"
    if name == "C3LE":
        assert int(r["n_draws"]) == 1
    if name == "C2N":
        assert int(r["counts"][3]) == 3 and int(r["n_ransac"]) == 2
        assert int(r["ransac0_num_inliers"]) == int(r["early_exit_min_inliers"]) - 1
    if name in ("C3L", "C3LT", "C3LE"):
        assert max(int(r["n_src"]), int(r["n_tgt"])) > 200000


# ------------------------------------------------------------------------------------------------ mutations
def _shared_sub(O, monkeypatch):
    """One sub-sample for every scale (the port's behaviour before the per-scale draw)."""
    est, cache = O.radius_estimation, {}

    def mut(src, skp, tgt, tkp, thresholds, tolerance=0.01, cum=None, sub_idx=None):
        n = max(len(src), len(tgt))
        if n > 200000 and sub_idx is None:
            if n not in cache:
                cache[n] = torch.randint(0, len(src) if len(src) > len(tgt) else len(tgt), (200000,)).numpy()
            sub_idx = cache[n]
        return est(src, skp, tgt, tkp, thresholds, tolerance, cum, sub_idx)

    monkeypatch.setattr(O, "radius_estimation", mut)


def _choose(pick_src):
    def mutation(O, monkeypatch):
        est = O.radius_estimation

        def mut(src, skp, tgt, tkp, thresholds, tolerance=0.01, cum=None, sub_idx=None):
            pts, kpts = (src, skp) if pick_src(len(src), len(tgt)) else (tgt, tkp)
            return est(pts, kpts, pts[:0], kpts, thresholds, tolerance, None, sub_idx)     # the chosen cloud alone

        monkeypatch.setattr(O, "radius_estimation", mut)

    return mutation


def _smaller_cloud(O, monkeypatch):
    """The smaller cloud sub-sampled (a tie still to the target)."""
    _choose(lambda ns, nt: ns < nt)(O, monkeypatch)


def _tie_to_source(O, monkeypatch):
    """A tie going to the source (the larger cloud otherwise)."""
    _choose(lambda ns, nt: ns >= nt)(O, monkeypatch)


def _no_rewind(O, monkeypatch):
    """All S sub-samples drawn before scale 0, none given back when the pair exits."""
    est, queue = O.radius_estimation, []

    def mut(src, skp, tgt, tkp, thresholds, tolerance=0.01, cum=None, sub_idx=None):
        n = len(src) if len(src) > len(tgt) else len(tgt)
        if n > 200000 and sub_idx is None:
            if not queue:
                queue.extend(torch.randint(0, n, (200000,)).numpy() for _ in range(3))
            sub_idx = queue.pop(0)
        return est(src, skp, tgt, tkp, thresholds, tolerance, cum, sub_idx)

    monkeypatch.setattr(O, "radius_estimation", mut)


def _exit_gt(O, monkeypatch):
    """`>` for `>=` in the early-exit test."""
    monkeypatch.setattr(O, "should_exit", lambda cfg, n: n > cfg.match.get("early_exit_min_inliers", 15))


def _aligned_lrf(O, monkeypatch):
    """The aligned route building the local reference frame anyway."""
    lrf = O.lrf
    monkeypatch.setattr(O, "lrf", lambda patches, des_r, aligned, *a, **kw: lrf(patches, des_r, False, *a, **kw))


MUTATIONS = [(_shared_sub, "C3L", 0), (_shared_sub, "C3LT", 0), (_smaller_cloud, "C3L", 0), (_tie_to_source, "C3LT", 0),
             (_no_rewind, "C3LE", 0), (_exit_gt, "C2E", 0), (_exit_gt, "C3LE", 0), (_aligned_lrf, "C3", 0),
             (_aligned_lrf, "C5", 0)]


@pytest.mark.parametrize("mutation,name,seed", MUTATIONS, ids=[f"{m.__name__[1:]}-{n}" for m, n, _ in MUTATIONS])
def test_route_pin_rejects_mutated_oracle(oracle, monkeypatch, mutation, name, seed):
    mutation(oracle, monkeypatch)
    out, draws = _replay(oracle, name, seed)
    monkeypatch.undo()
    with pytest.raises(AssertionError):
        _check(name, seed, out, draws)
