"""The local reference frame (a4+a5) against float64 without a GPU: oracle.lrf (bit-identical to the kernel,
tests/test_lrf_fp64_gpu.py) held patch by patch to oracle.lrf_fp64 on the hand-built edge patches (oracle/lrf_cases.py) and
on real C1 / C2 patches, in both Rodrigues forms; and the reference's own z axes (tests/golden/c2_seed*_reference.npz)
against float64 on the patches of those runs.

The bounds (oracle.lrf_cases.check_lrf; u = 2^-24; lam_1 <= lam_2 <= lam_3 the eigenvalues of the float64 covariance C of
the fp32 points about the key point c, gap = lam_2 - lam_1):

* z.  The fp32 covariance is C + E with |E| a small multiple of u lam_3 (fp32 products and sums of at most P / 32 + 5
  terms per lane and butterfly; p - c is exact for nearby points); the fp64 Jacobi adds nothing at that scale once it has
  converged (3 sweeps, 8 run).  First-order perturbation of the eigenvector of lam_1 gives angle <= |E| / gap, so
  angle(z, z64) <= b_z = KZ u lam_3 / gap.  Measured: 1.3 u lam_3 / gap on the edge cases and C1 / C2 (ratio 0.16).  Where b_z >
  1e-2 (near-degenerate, rank-deficient or zero covariance) z is not determined by C and only the backward statement is
  checked: z is an exact eigenvector of C + E for its smallest eigenvalue mu <= lam_1 + |E| (Weyl), so |C z| <= lam_1 +
  KZ u lam_3.  The angle is atan2(|a x b|, |a . b|) on normalised vectors: sqrt(1 - cos^2) reports a false 2.5e-4 because
  the fp32 z is not unit to fp64 precision.
* Sign.  The kernel flips z when fl(-z . c) < 0 on its fp32 z: that can differ from float64 only if |z64 . c| <=
  (b_z + KS u) |c|_1 (the z error plus the rounding of a three-term fp32 sum).  Outside that margin the signs must agree;
  inside it the float64 axis is taken on the kernel's side for the checks below.
* theta.  The kernel's cosine is fl(z_z / |z|) with |z_z - z64_z| <= eps_c = b_z sn + b_z^2 / 2 + KR u (a rotation by
  <= b_z moves cos(theta) by <= sin(theta) b_z + b_z^2 / 2), sn = |z64 x e_z|.  Literal form: theta = fl(acos(ct)) for
  an fp32 ct in [z64_z - eps_c, z64_z + eps_c]; acos is monotone, so the error is at most dtheta = max |acos(ct') -
  acos(z64_z)| over the two fp32 values that enclose that interval, + 2 pi u (rounding of theta, sin and cos).  Near
  |z_z| = 1 this is the acos step sqrt(2 u) = 3.45e-4 of the reference's formula, not a kernel fault.  Stable form:
  dtheta = b_z + KR u.
* R.  R depends on theta (|dR/dtheta| <= 1 entrywise) and on the axis a = (z_1, -z_0) / sn, whose error is da <=
  2 (b_z + KR u) / sn (a perturbation e of a vector v moves v / |v| by <= 2 |e| / |v|); the entries carry a times
  sin(theta) and (1 - cos(theta)), so |R - R64| <= dtheta + (2 (1 - cos theta) + sin theta) da + KR u entrywise.  Near
  theta = pi the axis term grows as 1 / sn and where the bound exceeds 1e-2 it says nothing: there the invariants are
  checked instead -- R R^T = I and det R = 1 to KO u, |R z64 - e_z| <= b_z + dtheta + KR u -- and R = I exactly where the
  axis is zero (z = +-e_z exactly; the kernel returns I at sn < 1e-12 like the reference's RodsRotatFormula).  A zero
  axis is only right for a vertical z: it needs z_0 = z_1 = 0 exactly (z_0 / 1e-12 cannot underflow), so its z is the
  line e_z, which is held to float64's by the z check like any other (sn64 <= b_z), and a supplied z must have z_0 = z_1
  = 0 there.  An identity frame on a patch whose float64 z is off the vertical fails.
* delta.  delta = fl(fl(R fl(p - c)) / r): against the kernel's own R applied in float64, |delta - R x / r| <= KD u
  (|R| |x|) / r componentwise; against R64, <= (bound_R + KD u) |x|_1 / r where the R bound is elementwise.
* rand_axis.  (z_1, -z_0, 0) / sn: within da of float64, its last entry exactly 0.
* Aligned.  R = I and rand_axis = (1, 0, 0) exactly, delta within 2 ulps of (p - c) / r.

Every KAPPA is 8 (16 for orthonormality); the largest measured ratios (err / bound) are printed with -s and recorded in
DESIGN.md section 7.  The reference's own z axes come from fp32 BLAS and an fp32 SVD: KAPPA_REF below is measured on its
three C2 runs."""
import hashlib
import os

import numpy as np
import pytest

from oracle import lrf_cases as L
from oracle.lrf_cases import merge, report

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
KAPPA_REF = 16.0          # reference z axes: angle <= KAPPA_REF u lam_3 / gap (measured ratio printed)

CASES = [(1, 0.5), (2, 0.5), (31, 0.02), (32, 50.0), (33, 1.0), (512, 0.02), (512, 1.0), (512, 50.0), (1000, 1.0)]


def run_oracle(oracle, monkeypatch, patches, des_r, aligned, stable):
    monkeypatch.setenv("BX_LRF", "stable" if stable else "literal")
    delta, Rt, ra, z = oracle.lrf(patches, des_r, aligned, want_z=True)
    out = L.check_lrf(patches, des_r, aligned, stable, delta, Rt, ra, z=None if aligned else z)
    if not aligned:     # z read back from R (what the GPU test sees) meets its own, wider bound
        out["z_from_R"] = L.check_lrf(patches, des_r, aligned, stable, delta, Rt, ra).get("z", 0.0)
    return out, z, Rt


@pytest.mark.parametrize("P,r", CASES, ids=[f"P{p}-r{r:g}" for p, r in CASES])
def test_lrf_fp64_against_the_oracle_on_edge_patches(oracle, monkeypatch, P, r):
    pat, lab = L.lrf_patches(P, r, seed=P)
    acc = {}
    for stable in (False, True):
        for aligned in (True, False):
            out, z, Rt = run_oracle(oracle, monkeypatch, pat, r, aligned, stable)
            merge(acc, out)
        # the zero covariance: the kernel's Jacobi leaves V = I and takes column 0, then the sign rule
        c = pat[:, -1].astype(np.float64)
        zero = (pat == pat[:, -1:]).all(axis=(1, 2))
        want = np.where(c[:, :1] > 0, -1.0, 1.0) * np.array([1.0, 0.0, 0.0])
        assert (z[zero] == want[zero]).all()
        assert (oracle.lrf_fp64(pat, r, False)["z"][zero] == want[zero]).all()
    # the regimes are there
    assert acc["z_eigenspace_n"] > 0
    if P >= 31:
        assert acc["R_identity"] > 0 and acc["z_angular"] > 0 and acc["R_elementwise_n"] > 0 and acc["R_invariants_n"] > 0 and acc["sign_checked"] > 0
        assert {"horizontal_above", "tilted_below", "octahedron", "empty_ball", "offset_plane"} <= set(lab)
    report(f"edge patches P={P} r={r:g} ({len(pat)} patches, both forms, both aligned flags)", acc)


@pytest.fixture(scope="module")
def c2_patches(oracle):
    """The oracle's patches of the three C2 reference runs, rebuilt from the golden key points (s_fps / t_fps), radii and
    permutations: per (seed, scale, side) the patches [1500,512,3], the radius and the reference's z axes.  The index rows
    hash to the golden s{i}_{side}_idx_sha, so these are the patches of those runs."""
    from bufferx_b200.synth import make_pair, workload_cfg
    cfg = workload_cfg("C2")
    K, P = cfg.patch.num_fps, cfg.patch.num_points_per_patch
    out = []
    for seed in (0, 1, 2):
        g = np.load(f"{ROOT}/tests/golden/c2_seed{seed}.npz")
        ref = np.load(f"{ROOT}/tests/golden/c2_seed{seed}_reference.npz")
        data = make_pair("C2", seed)
        perms = oracle.draw_perms(cfg, data["src_fds_pcd"].shape[0], data["tgt_fds_pcd"].shape[0], seed)
        for i in range(cfg.patch.num_scales):
            for j, (side, key, fk) in enumerate((("src", "src_fds_pcd", "s_fps"), ("tgt", "tgt_fds_pcd", "t_fps"))):
                pts = np.ascontiguousarray(data[key], dtype=np.float32)
                idx, pat = oracle.select_patches(pts, perms[i][j], pts[g[fk][:K]], float(g["des_r"][i]), P)
                sha = hashlib.sha256(np.ascontiguousarray(idx).tobytes()).hexdigest()[:16]
                assert sha == bytes(g[f"s{i}_{side}_idx_sha"]).decode(), f"seed {seed} scale {i} {side}: not the golden patches"
                out.append(dict(tag=f"seed{seed} s{i} {side}", patches=pat, des_r=float(g["des_r"][i]), z_ref=ref[f"s{i}_{side}_z"]))
    return out


def test_lrf_fp64_against_the_oracle_on_c1_c2_patches(oracle, monkeypatch, c1, c2_patches):
    """Real patches: the C1 pair's three scales (src and tgt) and the C2 seed-0 pair's six (cloud, scale) sets, 9000."""
    sets = [(f"C1 s{i} {side}", sc[side]["patches"], c1["res"][5]["des_r"][i])
            for i, sc in enumerate(c1["res"][5]["scales"]) for side in ("src", "tgt")]
    sets += [(d["tag"], d["patches"], d["des_r"]) for d in c2_patches if d["tag"].startswith("seed0")]
    for stable in (False, True):
        acc = {}
        for tag, pat, r in sets:
            merge(acc, run_oracle(oracle, monkeypatch, pat, r, False, stable)[0])
        report(f"C1 + C2 patches, {'stable' if stable else 'literal'} form", acc)


def test_reference_z_axes_against_fp64(oracle, c2_patches):
    """The z axes the reference's own forward handed to RodsRotatFormula (three C2 runs, 27000 patches; its covariance is
    an fp32 BLAS product and its eigenvector an fp32 SVD) against float64 on the same patches: angle <= KAPPA_REF u lam_3 /
    gap where that is below 1e-2, no sign flip outside the rounding margin, and the oracle's own axes within KZ."""
    worst_ref, worst_own, deg_max, flips, checked, n = 0.0, 0.0, 0.0, 0, 0, 0
    for d in c2_patches:
        ref = oracle.lrf_fp64(d["patches"], d["des_r"], False)
        zr = d["z_ref"].astype(np.float64)
        _, _, _, zo = oracle.lrf(d["patches"], d["des_r"], False, want_z=True)
        b = np.where(ref["gap"] > 0, U * ref["lam"][:, 2] / np.where(ref["gap"] > 0, ref["gap"], 1), np.inf)
        ok = b * KAPPA_REF <= 1e-2
        a = L.angle(zr, ref["z"])
        worst_ref = max(worst_ref, float((a[ok] / b[ok]).max()))
        assert (a[ok] <= KAPPA_REF * b[ok]).all(), f"{d['tag']}: reference z beyond {KAPPA_REF} u lam_3 / gap"
        deg_max = max(deg_max, float(np.degrees(a).max()))
        worst_own = max(worst_own, float((L.angle(zo.astype(np.float64), ref["z"])[ok] / b[ok]).max()))
        c = d["patches"][:, -1].astype(np.float64)
        clear = ok & (ref["margin"] > (KAPPA_REF * b + L.KS * U) * np.abs(c).sum(axis=1))
        flips += int((clear & (np.einsum("ki,ki->k", zr, ref["z"]) < 0)).sum())
        checked += int(clear.sum())
        n += len(zr)
    assert flips == 0, f"{flips} sign flips of the reference's z against float64"
    assert worst_own <= L.KZ
    print(f"\n[lrf-fp64] reference z axes, {n} patches: angle / (u lam_3 / gap) max {worst_ref:.3g} (KAPPA_REF {KAPPA_REF:g}); "
          f"largest angle {deg_max:.3g} deg; {checked} signs checked, 0 flips; the oracle's own axes {worst_own:.3g}")
