"""The local reference frame (a4+a5) on the GPU against float64, on edge patches and on the route production runs.

bx_lrf_batched is held bit for bit to oracle.lrf (same fp32 operation order, -fmad=false) and, patch by patch, to the
float64 bounds of oracle.lrf_cases.check_lrf, derived in the docstring of tests/test_lrf_fp64_cpu.py: the z axis (third
column of Rt) within KZ u lam_3 / gap of float64's -- plus the acos error of theta in the literal form, since R's third
row is rebuilt from theta -- or in the near-null eigenspace where the spectrum does not determine it; the sign rule equal
to float64's outside the rounding margin; R elementwise, or its invariants where the elementwise bound is vacuous
(theta near pi); R = I where the axis is zero, whose z (the line e_z) is then held to float64's; delta against the
kernel's own R and against float64's; rand_axis; the aligned path exact.  Both Rodrigues forms (BX_LRF=stable is read on every call by ops.lrf and oracle.lrf).

Routes: ops.lrf with one host radius (MiniSpinNet.forward), device radii with r_group (one launch over every patch of a
pair, patch k uses radii[k // r_group]) and MiniSpinNet.forward_multi with ``radii`` on the C2 seed-0 pair, 9000 patches
in that single launch.  The largest ratio of each check is printed (run with -s) and recorded in DESIGN.md section 7."""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import lrf_cases as L
from oracle.lrf_cases import merge, report

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = [(1, 0.5), (2, 0.5), (31, 0.02), (32, 50.0), (33, 1.0), (512, 0.02), (512, 1.0), (512, 50.0), (1000, 1.0)]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


def cu(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def bits_equal(name, got, want):
    got = got.cpu().numpy() if isinstance(got, torch.Tensor) else got
    bad = got.view(np.int32) != np.asarray(want, np.float32).view(np.int32)
    assert not bad.any(), f"{name}: {int(bad.sum())} values differ from the oracle, first at {np.argwhere(bad)[:3].tolist()}"


def gpu_vs_oracle(oracle, dev, patches, des_r, aligned):
    """ops.lrf and oracle.lrf on the same patches (one host radius): bit for bit -> the GPU outputs (numpy)."""
    from bufferx_b200 import ops
    d, Rt, ra = ops.lrf(cu(patches, dev), des_r, aligned)
    ed, eR, era = oracle.lrf(patches, des_r, aligned)
    for name, a, b in (("delta", d, ed), ("Rt", Rt, eR), ("rand_axis", ra, era)):
        bits_equal(name, a, b)
    return d.cpu().numpy(), Rt.cpu().numpy(), ra.cpu().numpy()


@pytest.mark.parametrize("P,r", CASES, ids=[f"P{p}-r{r:g}" for p, r in CASES])
def test_lrf_edge_patches(dev, oracle, monkeypatch, P, r):
    """The hand-built edge patches (oracle/lrf_cases.py): both Rodrigues forms, both aligned flags."""
    pat, _ = L.lrf_patches(P, r, seed=P)
    acc = {}
    for stable in (False, True):
        monkeypatch.setenv("BX_LRF", "stable" if stable else "literal")
        for aligned in (False, True):
            d, Rt, ra = gpu_vs_oracle(oracle, dev, pat, r, aligned)
            merge(acc, L.check_lrf(pat, r, aligned, stable, d, Rt, ra))
    report(f"edge patches P={P} r={r:g}: bit-exact to the oracle", acc)


@pytest.mark.parametrize("K", [0, 1, 3, 5, 4097])
@pytest.mark.parametrize("P", [33, 512])
def test_lrf_patch_counts(dev, oracle, monkeypatch, K, P):
    """K not a multiple of the 4 patches of a CTA, K = 0 (no launch) and K = 4097 (the edge patches tiled)."""
    pat, _ = L.lrf_patches(P, 1.0, seed=P + 1)
    pat = np.ascontiguousarray(pat[np.arange(K) % len(pat)]).reshape(K, P, 3)
    acc = {}
    for stable in (False, True):
        monkeypatch.setenv("BX_LRF", "stable" if stable else "literal")
        for aligned in (False, True):
            d, Rt, ra = gpu_vs_oracle(oracle, dev, pat, 1.0, aligned)
            assert d.shape == (K, P, 3) and Rt.shape == (K, 3, 3) and ra.shape == (K, 3)
            merge(acc, L.check_lrf(pat, 1.0, aligned, stable, d, Rt, ra))
    report(f"K={K} P={P}", acc)


@pytest.mark.parametrize("G", [1, 7, 33])
def test_lrf_device_radii_r_group(dev, oracle, monkeypatch, G):
    """Device radii [0.5, 1, 2] with r_group = G in {1, 7, 33} (not multiples of 4): patch k uses radii[k // G], so
    a wrong group index moves delta by a factor of 2 or more.  Into caller-owned NaN-filled buffers with two spare rows:
    bit for bit against one host-radius call per group, within the float64 bounds at the per-patch radius, rows past K
    untouched."""
    from bufferx_b200 import ops
    radii = np.array([0.5, 1.0, 2.0], np.float32)
    P = 64
    pat, _ = L.lrf_patches(P, 1.0, seed=G)
    K = 3 * G
    pat = np.ascontiguousarray(pat[np.arange(K) % len(pat)])
    rk = radii[np.arange(K) // G]
    acc = {}
    for stable in (False, True):
        monkeypatch.setenv("BX_LRF", "stable" if stable else "literal")
        for aligned in (False, True):
            d = torch.full((K + 2, P, 3), float("nan"), device=dev)
            Rt = torch.full((K + 2, 3, 3), float("nan"), device=dev)
            ra = torch.full((K + 2, 3), float("nan"), device=dev)
            ops.lrf(cu(pat, dev), cu(radii, dev), aligned, delta=d[:K], Rt=Rt[:K], ra=ra[:K], r_group=G)
            assert torch.isnan(d[K:]).all() and torch.isnan(Rt[K:]).all() and torch.isnan(ra[K:]).all(), "rows past K written"
            for g in range(3):
                s = slice(g * G, (g + 1) * G)
                gd, gR, ga = ops.lrf(cu(pat[s], dev), float(radii[g]), aligned)
                bits_equal(f"group {g} delta", d[s], gd.cpu().numpy())
                bits_equal(f"group {g} Rt", Rt[s], gR.cpu().numpy())
                bits_equal(f"group {g} rand_axis", ra[s], ga.cpu().numpy())
            merge(acc, L.check_lrf(pat, rk, aligned, stable, d[:K].cpu().numpy(), Rt[:K].cpu().numpy(), ra[:K].cpu().numpy()))
    report(f"device radii, r_group={G}", acc)


def test_lrf_forward_multi_c2_pair(dev, oracle, monkeypatch):
    """The production route at production size: MiniSpinNet.forward_multi on the C2 seed-0 pair's six (cloud, scale) jobs
    with ``radii`` -- one bx_lrf_batched launch over 9000 patches, r_group = 3000 -- every row of R, delta and rand_axis
    against float64.  ops.lrf is wrapped to record that forward_multi made exactly that one call (the per-job route gives
    the same bits and would otherwise pass unnoticed).  The raw patches are gathered again with ops.select_patches
    (bit-identical to the batched gather); their index rows hash to the golden run's."""
    import bufferx_b200 as bx
    from bufferx_b200 import ops
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg
    monkeypatch.delenv("BX_LRF", raising=False)
    cfg = workload_cfg("C2")
    K, P, S = cfg.patch.num_fps, cfg.patch.num_points_per_patch, cfg.patch.num_scales
    g = np.load(f"{ROOT}/tests/golden/c2_seed0.npz")
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True).to(dev).eval()
    data = make_pair("C2", 0)
    aligned = bool(data["is_aligned_to_global_z"])
    assert not aligned
    perms = oracle.draw_perms(cfg, data["src_fds_pcd"].shape[0], data["tgt_fds_pcd"].shape[0], 0)
    radii = cu(g["des_r"].astype(np.float32), dev)
    jobs, raw = [], []
    for i in range(S):
        for j, (side, key, fk) in enumerate((("src", "src_fds_pcd", "s_fps"), ("tgt", "tgt_fds_pcd", "t_fps"))):
            pts = np.ascontiguousarray(data[key], dtype=np.float32)
            job = (cu(pts, dev), cu(pts[g[fk][:K]], dev), radii[i:i + 1], cu(perms[i][j].astype(np.int32), dev))
            jobs.append(job)
            pat, idx = ops.select_patches(ops.permute_cloud(job[0], job[3]), job[1], job[2], P, want_idx=True)
            sha = hashlib.sha256(np.ascontiguousarray(idx.cpu().numpy()).tobytes()).hexdigest()[:16]
            assert sha == bytes(g[f"s{i}_{side}_idx_sha"]).decode(), f"scale {i} {side}: not the golden patches"
            raw.append(pat.cpu().numpy())
    calls = []
    lrf = ops.lrf

    def recording_lrf(patches, des_r, *a, **kw):
        calls.append((patches.shape[0], isinstance(des_r, torch.Tensor), kw.get("r_group", 0)))
        return lrf(patches, des_r, *a, **kw)

    monkeypatch.setattr(ops, "lrf", recording_lrf)
    with torch.no_grad():
        outs = model.Desc.forward_multi(jobs, aligned, radii=radii)
    monkeypatch.setattr(ops, "lrf", lrf)
    assert calls == [(2 * S * K, True, 2 * K)], f"forward_multi did not take the one-launch LRF route: {calls}"
    delta = torch.cat([o["patches"] for o in outs]).cpu().numpy()
    Rt = model.Desc.last_multi["R"].cpu().numpy()
    ra = torch.cat([o["rand_axis"] for o in outs]).cpu().numpy()
    raw = np.concatenate(raw)
    assert delta.shape == (2 * S * K, P, 3) == raw.shape
    for n in range(2 * S):
        s = slice(n * K, (n + 1) * K)
        ed, eR, era = oracle.lrf(raw[s], float(g["des_r"][n // 2]), aligned)
        bits_equal(f"job {n} delta", delta[s], ed)
        bits_equal(f"job {n} Rt", Rt[s], eR)
        bits_equal(f"job {n} rand_axis", ra[s], era)
    rk = np.repeat(g["des_r"].astype(np.float32), 2 * K)
    out = L.check_lrf(raw, rk, aligned, False, delta, Rt, ra)
    report("forward_multi C2 seed 0, 9000 patches in one launch: bit-exact to the oracle", out)
