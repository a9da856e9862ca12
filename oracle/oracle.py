"""CPU ORACLE of the BUFFER-X per-pair registration hot path (python side).

TEST INFRASTRUCTURE ONLY -- imported by tests/, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py``; the product package
(``buffer-x_b200/``) never imports it.

PARITY STATUS: "parity unpinned" by the reference's own tests (it has none, SURVEY.md
section 4).  What pins this oracle instead is ``oracle/ref_check.py``: it imports the
reference's own Python from /root/reference in the build container, runs its
``BufferX.forward`` on CPU with the missing third-party leaf ops (pointnet2_ops, knn_cuda,
torch_batch_svd, kornia, open3d) provided by the restatements below, compares every stage
with this pipeline and writes ``tests/golden/*.npz``.

Stages (ids of SURVEY.md section 8a; file:line are relative to /root/reference):
    a1  fps                      models/BUFFERX.py:286-290, 338-346 (pointnet2_ops, not vendored)
    a2  radius_estimation        models/BUFFERX.py:610-696
    a3  select_patches           models/patch_embedder.py:92-120
    a4  lrf (axis_align)         models/patch_embedder.py:122-148, utils/common.py:501-525, 709-726
    a5  normalize                models/patch_embedder.py:167-170
    a6  spt                      models/patch_embedder.py:150-165, utils/common.py:422-498
    a7  pnt_layer + max          models/patch_embedder.py:26-30, 73-77
    a8  cylindrical conv net     models/patchnet.py:16-84, utils/common.py:265-310
    a9  attention pooling        models/patch_embedder.py:32-39, 80-83
    a10 mutual matching          models/BUFFERX.py:469-496 (knn_cuda, not vendored)
    a11 cost volume + CostNet    models/BUFFERX.py:39-69, models/patchnet.py:151-210
    a12 hypothesis build         models/BUFFERX.py:382-389 (kornia Rodrigues)
    a13 consensus                models/BUFFERX.py:392-417
    a14 RANSAC                   models/pose_estimator.py:84-117 (Open3D 0.18, not vendored)
    a15 post refinement          models/BUFFERX.py:522-603
Integer / index stages are evaluated by the C file ``oracle/c/bx_oracle.c`` with a frozen
fp32 operation order; the conv stacks use torch CPU fp32 (tolerance parity, 1e-4 rel).
"""
from __future__ import annotations

import ctypes
import math
import os
import subprocess
import time
from ctypes import POINTER, c_double, c_float, c_int, c_int32, c_int64, c_uint64, c_void_p

import numpy as np
import torch
import torch.nn.functional as F

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liboracle.so")
_SRC = os.path.join(_HERE, "c", "bx_oracle.c")


def build(force: bool = False) -> str:
    """Compile the C restatement (gcc, no FMA contraction, OpenMP)."""
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        cmd = ["gcc", "-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fno-fast-math",
               "-fvisibility=hidden", "-std=c11", "-o", _SO, _SRC, "-lm"]
        subprocess.check_call(cmd)
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(build())
        _lib.bxo_ransac.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_double, c_double, c_double, c_int,
                                    c_uint64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
        _lib.bxo_radius_bisect.argtypes = [c_void_p, c_int64, c_double, c_double]
        _lib.bxo_radius_bisect.restype = c_int
        _lib.bxo_ball_query.argtypes = [c_void_p, c_int, c_void_p, c_int, c_float, c_int, c_void_p, c_void_p]
        _lib.bxo_select_patches.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_int, c_float, c_int, c_void_p, c_void_p]
        _lib.bxo_lrf.argtypes = [c_void_p, c_int, c_int, c_float, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
        _lib.bxo_spt.argtypes = [c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p, c_float, c_int, c_void_p, c_void_p]
        _lib.bxo_consensus.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p]
        _lib.bxo_refine.argtypes = [c_void_p, c_void_p, c_int, c_void_p, c_float, c_void_p, c_void_p]
        _lib.bxo_horn_fit.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_double, c_void_p]
        _lib.bxo_fps.argtypes = [c_void_p, c_int, c_int, c_void_p]
        _lib.bxo_mutual_nn.argtypes = [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]
        _lib.bxo_radius_hist.argtypes = [c_void_p, c_int, c_void_p, c_int, c_void_p]
    return _lib


def _p(a):
    return a.ctypes.data_as(c_void_p) if a is not None else None


def _f32(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32))


def num_threads() -> int:
    return int(lib().bxo_num_threads())


# --------------------------------------------------------------------------- #
# integer / index stages (C)
# --------------------------------------------------------------------------- #
def fps(xyz, npoint: int) -> np.ndarray:
    xyz = _f32(xyz)
    idx = np.zeros(npoint, dtype=np.int32)
    rc = lib().bxo_fps(_p(xyz), xyz.shape[0], npoint, _p(idx))
    assert rc == 0
    return idx


def ball_query(xyz, qry, radius: float, nsample: int):
    xyz, qry = _f32(xyz), _f32(qry)
    idx = np.zeros((qry.shape[0], nsample), dtype=np.int32)
    cnt = np.zeros(qry.shape[0], dtype=np.int32)
    lib().bxo_ball_query(_p(xyz), xyz.shape[0], _p(qry), qry.shape[0], c_float(radius), nsample, _p(idx), _p(cnt))
    return idx, cnt


def select_patches(pts, perm, kpts, radius: float, P: int):
    pts, kpts = _f32(pts), _f32(kpts)
    perm = None if perm is None else np.ascontiguousarray(perm, dtype=np.int32)
    K = kpts.shape[0]
    idx = np.zeros((K, P), dtype=np.int32)
    patches = np.zeros((K, P, 3), dtype=np.float32)
    rc = lib().bxo_select_patches(_p(pts), pts.shape[0], _p(perm), _p(kpts), K, c_float(radius), P, _p(idx), _p(patches))
    assert rc == 0
    return idx, patches


def lrf_stable() -> bool:
    """BX_LRF=stable selects the well-conditioned Rodrigues form (not the reference's; sensitivity studies only)."""
    return os.environ.get("BX_LRF", "").lower() == "stable"


def lrf(patches, des_r: float, aligned: bool, z_axis=None, want_z=False):
    """a4+a5.  ``z_axis`` [K,3]: use these (disambiguated, unit) axes instead of the covariance/Jacobi result."""
    patches = _f32(patches)
    K, P, _ = patches.shape
    delta = np.zeros_like(patches)
    Rt = np.zeros((K, 3, 3), dtype=np.float32)
    ra = np.zeros((K, 3), dtype=np.float32)
    zo = None if z_axis is None else _f32(z_axis)
    z_out = np.zeros((K, 3), dtype=np.float32)
    flags = int(bool(aligned)) | (2 if lrf_stable() else 0)
    lib().bxo_lrf(_p(patches), K, P, c_float(des_r), flags, _p(delta), _p(Rt), _p(ra), _p(zo), _p(z_out))
    if want_z:
        return delta, Rt, ra, z_out
    return delta, Rt, ra


def rodrigues_fp64(z, stable=False):
    """The rotation of ``lrf`` taking unit z [K,3] (float64) onto +e_z, evaluated in float64 -> (R [K,3,3], rand_axis
    [K,3]).  theta = arccos(z_z) (the literal form) or cos = z_z, sin = |z x e_z| (stable); axis a = (z_1, -z_0) /
    max(sn, 1e-12) with sn = |z x e_z|, R = I + sin [a]x + (1 - cos) [a]x^2 written out like the kernel, so that sn = 0
    gives R = I."""
    z = np.asarray(z, dtype=np.float64)
    sn = np.hypot(z[:, 0], z[:, 1])
    if stable:
        ct, st = z[:, 2], sn
    else:
        th = np.arccos(np.clip(z[:, 2], -1.0, 1.0))
        ct, st = np.cos(th), np.sin(th)
    den = np.maximum(sn, 1e-12)
    a0, a1 = z[:, 1] / den, -z[:, 0] / den
    kk = 1.0 - ct
    R = np.empty((len(z), 3, 3))
    R[:, 0, 0], R[:, 0, 1], R[:, 0, 2] = 1.0 - kk * a1 * a1, kk * a0 * a1, st * a1
    R[:, 1, 0], R[:, 1, 1], R[:, 1, 2] = kk * a0 * a1, 1.0 - kk * a0 * a0, -st * a0
    R[:, 2, 0], R[:, 2, 1], R[:, 2, 2] = -st * a1, st * a0, 1.0 - kk * (a0 * a0 + a1 * a1)
    return R, np.stack([a0, a1, np.zeros_like(a0)], axis=1)


def lrf_fp64(patches, des_r, aligned: bool, stable: bool = False):
    """a4+a5 in float64 on the fp32 patches [K,P,3] (key point last): the covariance of p - c about the key point c,
    numpy's eigh and its eigenvector of the smallest eigenvalue, the sign rule of ``lrf`` (flip when -z . c < 0), then
    ``rodrigues_fp64`` and delta = R (p - c) / r.  ``des_r``: a scalar or one radius per patch, used at its fp32 value (the
    value the kernel divides by).  An all-zero covariance gets e_x before the sign rule, the choice of the kernel's
    Jacobi (no rotation, first minimum); the reference leaves it open.
    -> dict(C, lam (ascending), gap = lam_2 - lam_1, z (sign ruled, unit), margin = |z . c|, sn = |z x e_z|, R (applied to
    delta, R z = e_z), Rt (the transpose, what ``lrf`` returns), rand_axis, delta), float64 throughout."""
    pt = np.asarray(patches, dtype=np.float32).astype(np.float64)
    K = pt.shape[0]
    c = pt[:, -1, :]
    d = pt - c[:, None, :]
    r = np.broadcast_to(np.asarray(des_r, dtype=np.float32).astype(np.float64), (K,))
    C = np.einsum("kpi,kpj->kij", d, d)
    lam, V = np.linalg.eigh(C) if K else (np.zeros((0, 3)), np.zeros((0, 3, 3)))
    z = V[:, :, 0].copy()
    zero = ~C.reshape(K, 9).any(axis=1)
    z[zero] = (1.0, 0.0, 0.0)
    dot = np.einsum("ki,ki->k", z, c)
    z[-dot < 0] *= -1.0
    if aligned:
        R, ra = np.broadcast_to(np.eye(3), (K, 3, 3)).copy(), np.broadcast_to([1.0, 0.0, 0.0], (K, 3)).copy()
    else:
        R, ra = rodrigues_fp64(z, stable)
    delta = np.einsum("kij,kpj->kpi", R, d) / r[:, None, None]
    return dict(C=C, lam=lam, gap=lam[:, 1] - lam[:, 0], z=z, margin=np.abs(dot), sn=np.hypot(z[:, 0], z[:, 1]), R=R,
                Rt=R.transpose(0, 2, 1).copy(), rand_axis=ra, delta=delta)


def voxel_table(rad_n=3, azi_n=20, ele_n=7) -> np.ndarray:
    """[rad_n*ele_n*azi_n, 3] fp32 voxel centres, built in fp64 exactly like
    ``utils/common.py:248-262, 392-405, 422-428`` (s2_grid -> change_coordinates -> shell scale)."""
    beta = np.linspace(0, np.pi, num=ele_n, endpoint=False) + np.pi / ele_n / 2
    alpha = np.linspace(0, 2 * np.pi, num=azi_n, endpoint=False) + np.pi / azi_n
    B, A = np.meshgrid(beta, alpha, indexing="ij")
    B, A = B.flatten(), A.flatten()
    r = 1  # SPT is called with des_r = 1 (patch_embedder.py:70)
    xyz = np.stack([r * np.sin(B) * np.cos(A), r * np.sin(B) * np.sin(A), r * np.cos(B)], axis=1)
    xyz = np.repeat(xyz[None], rad_n, axis=0)
    scale = np.reshape(np.arange(rad_n) / rad_n + 1 / (2 * rad_n), [rad_n, 1, 1])
    return (scale * xyz).reshape(-1, 3).astype(np.float32)


def derot_table(azi_n=20) -> np.ndarray:
    """[azi_n, 2] fp32 (cos, sin) of -a*2pi/azi_n, fp64 then cast (``utils/common.py:483-491``)."""
    ang = -1.0 * np.arange(azi_n) * (2 * np.pi / azi_n)
    return np.stack([np.cos(ang), np.sin(ang)], axis=1).astype(np.float32)


def spt(delta, rad_n=3, azi_n=20, ele_n=7, voxel_r: float = 0.8 / 3, nv: int = 10):
    delta = _f32(delta)
    K, P, _ = delta.shape
    vox = voxel_table(rad_n, azi_n, ele_n)
    rot = derot_table(azi_n)
    V = vox.shape[0]
    out = np.zeros((K, V, nv, 3), dtype=np.float32)
    vidx = np.zeros((K, V, nv), dtype=np.int32)
    lib().bxo_spt(_p(delta), K, P, _p(vox), V, azi_n, _p(rot), c_float(voxel_r), nv, _p(out), _p(vidx))
    return out, vidx


def mutual_nn(a, b):
    a, b = _f32(a), _f32(b)
    Ka, Kb = a.shape[0], b.shape[0]
    s = np.zeros(max(Ka, 1), dtype=np.int32)
    t = np.zeros(max(Ka, 1), dtype=np.int32)
    snn = np.zeros(max(Ka, 1), dtype=np.int32)
    tnn = np.zeros(max(Kb, 1), dtype=np.int32)
    M = lib().bxo_mutual_nn(_p(a), Ka, _p(b), Kb, a.shape[1], _p(s), _p(t), _p(snn), _p(tnn))
    assert M >= 0
    return s[:M].copy(), t[:M].copy(), snn[:Ka], tnn[:Kb]


def radius_hist(kpts, pts) -> np.ndarray:
    kpts, pts = _f32(kpts), _f32(pts)
    cum = np.zeros(8193, dtype=np.int64)
    rc = lib().bxo_radius_hist(_p(kpts), kpts.shape[0], _p(pts), pts.shape[0], _p(cum))
    assert rc == 0
    return cum


def radius_estimation(src_pts, src_kpts, tgt_pts, tgt_kpts, thresholds, tolerance=0.01, cum=None, sub_idx=None):
    """``density_aware_radius_estimation`` (models/BUFFERX.py:627-696): the larger cloud wins
    (strict >, else target); returns the list of 2-decimal radii.  Above 200000 points the reference histograms
    ``pts[sub_idx]`` and keeps the original size in the denominator; without ``sub_idx`` this call makes the reference's
    draw itself, ``torch.randint(0, N, (200000,))`` from torch's CPU generator (the reference calls this function once per
    scale, so each scale draws its own sub-sample)."""
    if src_pts.shape[0] > tgt_pts.shape[0]:
        pts, kpts = src_pts, src_kpts
    else:
        pts, kpts = tgt_pts, tgt_kpts
    denom = int(pts.shape[0]) * int(kpts.shape[0])
    if pts.shape[0] > 200000:
        if sub_idx is None:
            sub_idx = torch.randint(0, pts.shape[0], (200000,)).numpy()
        pts = np.asarray(pts)[np.asarray(sub_idx)]
    if cum is None:
        cum = radius_hist(kpts, pts)
    out = []
    for th in thresholds:
        m = lib().bxo_radius_bisect(_p(cum), c_int64(denom), float(th), float(tolerance))
        out.append(round(5.0 * m / 8192.0, 2))
    return out


def consensus(ss, tt, R, t, azi_n: int, inlier_th: float):
    ss, tt, R, t = _f32(ss), _f32(tt), _f32(R), _f32(t)
    Mc = ss.shape[0]
    ind = np.zeros(max(Mc, 1), dtype=np.int32)
    best = np.zeros(1, dtype=np.int32)
    counts = np.zeros(max(Mc, 1), dtype=np.int32)
    I = lib().bxo_consensus(_p(ss), _p(tt), _p(R), _p(t), Mc, azi_n, c_float(inlier_th), _p(ind), _p(best), _p(counts))
    return ind[:I].copy(), int(best[0]), counts[:Mc]


class RansacRec(ctypes.Structure):
    _fields_ = [("pass_", c_int32), ("good", c_int32), ("rmse", c_double)]


def ransac(src, tgt, inlier_ind, dist_th, similar_th, confidence, max_iter, seed, want_recs=False):
    src, tgt = _f32(src), _f32(tgt)
    ind = np.ascontiguousarray(inlier_ind, dtype=np.int32)
    T = np.zeros(16, dtype=np.float64)
    ninl = np.zeros(1, dtype=np.int32)
    bitr = np.zeros(1, dtype=np.int32)
    iters = np.zeros(1, dtype=np.int32)
    recs = (RansacRec * max_iter)() if want_recs else None
    lib().bxo_ransac(_p(src), _p(tgt), _p(ind), len(ind), float(dist_th), float(similar_th), float(confidence),
                     int(max_iter), c_uint64(seed), _p(T), _p(ninl), _p(bitr), _p(iters),
                     ctypes.cast(recs, c_void_p) if recs is not None else None)
    out = dict(T=T.reshape(4, 4).copy(), num_inliers=int(ninl[0]), best_itr=int(bitr[0]), iters=int(iters[0]))
    if want_recs:
        n = int(iters[0])
        out["recs"] = np.array([(recs[i].pass_, recs[i].good, recs[i].rmse) for i in range(n)],
                               dtype=[("pass", "i4"), ("good", "i4"), ("rmse", "f8")])
    return out


def refine(src, tgt, T_in, dist_th):
    src, tgt = _f32(src), _f32(tgt)
    Tin = _f32(np.asarray(T_in).reshape(16))
    Tout = np.zeros(16, dtype=np.float32)
    rounds = np.zeros(1, dtype=np.int32)
    lib().bxo_refine(_p(src), _p(tgt), src.shape[0], _p(Tin), c_float(dist_th), _p(Tout), _p(rounds))
    return Tout.reshape(4, 4).copy(), int(rounds[0])


def horn_fit(a, b, w=None, eps=0.0):
    """The C restatement's rigid fit; ``eps`` is added to the weight sum of the centroids (refinement: 1e-6)."""
    a = np.ascontiguousarray(a, dtype=np.float64)
    b = np.ascontiguousarray(b, dtype=np.float64)
    w = None if w is None else np.ascontiguousarray(w, dtype=np.float64)
    T = np.zeros(16, dtype=np.float64)
    lib().bxo_horn_fit(_p(a), _p(b), _p(w), a.shape[0], c_double(eps), _p(T))
    return T.reshape(4, 4)


# --------------------------------------------------------------------------- #
# a1-a3 evaluated in float64 from the reference's formulas (tests/test_frontend_fp64_*.py).  Torch on whichever device
# the inputs live on; the fp32 inputs are widened exactly.  Margins use U = 2^-24; the bounds are derived in
# tests/test_frontend_fp64_cpu.py.
# --------------------------------------------------------------------------- #
U24 = 2.0 ** -24
RADIUS_MAX = 5.0
RADIUS_BINS = 8192


def _t64(a, device=None):
    t = a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    return t.to(device=device if device is not None else t.device, dtype=torch.float32).to(torch.float64)


def _fits32(v):
    """v (float64) is an fp32 value: the fp32 operation that produced it was exact."""
    return v.to(torch.float32).to(torch.float64) == v


def fps_fp64(xyz, idx, ks=4.0, kd=12.0):
    """pointnet2 ``furthest_point_sample`` in float64 on the fp32 coordinates, teacher-forced on the picks ``idx``.

    A point is skipped when mag = x*x+y*y+z*z <= 1e-3 (double literal); the skip is decided outside ks*u*1e-3 of it, or
    exactly when every fp32 partial sum of mag is exact.  temp = running minimum of the float64 distances to the earlier
    picks (from 1e10).  At step j the candidates are the points not decided-skipped; vmax = the largest temp of the
    decided-valid ones, margin = kd*u*vmax.  Returns per step j >= 1 (index j-1): vmax, the pick's temp, the largest
    decided-valid temp strictly below vmax (-1 if none), whether the pick is a candidate, whether the step is decided
    (vmax - second > margin and no undecided-skip point within the margin of vmax or above), and the number of
    decided-valid points."""
    x = _t64(xyz)
    idx = torch.as_tensor(np.asarray(idx) if not isinstance(idx, torch.Tensor) else idx).to(x.device).long()
    n, m = x.shape[0], idx.shape[0]
    sq = x * x
    s1 = sq[:, 0] + sq[:, 1]
    mag = s1 + sq[:, 2]
    exact = _fits32(sq).all(1) & _fits32(s1) & _fits32(mag)
    lo_m, hi_m = 1e-3 * (1 - ks * U24), 1e-3 * (1 + ks * U24)
    valid = torch.where(exact, mag > 1e-3, mag > hi_m)
    skip = torch.where(exact, mag <= 1e-3, mag < lo_m)
    cand = ~skip
    n_valid = int(valid.sum())
    temp = torch.full((n,), 1e10, dtype=torch.float64, device=x.device)
    steps = max(m - 1, 0)
    vmax = torch.zeros(steps, dtype=torch.float64, device=x.device)
    vpick, vsec = torch.zeros_like(vmax), torch.zeros_like(vmax)
    pick_ok = torch.zeros(steps, dtype=torch.bool, device=x.device)
    decided = torch.zeros_like(pick_ok)
    neg = torch.tensor(-1.0, dtype=torch.float64, device=x.device)
    for j in range(1, m):
        d = ((x - x[idx[j - 1]]) ** 2).sum(1)
        temp = torch.minimum(temp, d)
        t = torch.where(valid, temp, neg)
        mx = t.max()
        below = torch.where(t == mx, neg, t).max()
        und = torch.where(cand & ~valid, temp, neg).max()
        k = idx[j]
        vmax[j - 1], vsec[j - 1] = mx, below
        vpick[j - 1] = torch.where(cand[k], temp[k], neg)
        pick_ok[j - 1] = cand[k] | ((k == 0) & (n_valid == 0))
        marg = kd * U24 * mx
        decided[j - 1] = (mx - below > marg) & (und < mx - marg)
    return dict(vmax=vmax, vpick=vpick, vsecond=vsec, pick_ok=pick_ok, decided=decided, n_valid=n_valid,
                n_skip=int(skip.sum()), n_undecided_skip=int((~valid & ~skip).sum()))


def radius_count_bounds(kpts, pts, kc=9.0, chunk=1 << 23):
    """squared_cdist (BUFFERX.py:610-624) as count intervals over the 8193 probed radii r_m = 5 m / 8192.

    d64 = |k - p|^2; the reference's (|k|^2 + |p|^2) - 2 k.p in fp32 (any order, FMA or not) lies within
    e = kc*u*(|k|^2 + |p|^2) of it -- and equals it when every coordinate is a multiple of 2^-13 and (|k| + |p|)^2 < 1/4
    (every partial sum is then a multiple of 2^-26 below 2^-2: exact in fp32).  The filter d2 <= max_r^2 keeps every d2
    below a probed threshold, so it never changes a count.  Returns (lo, hi) int64 [8193]:
    lo[m] = #{d64 + e < thr_m} <= count(m) <= hi[m] = #{d64 - e < thr_m}, thr_m = fl32(r_m^2)."""
    k, p = _t64(kpts), _t64(pts)
    dev = k.device
    m = torch.arange(RADIUS_BINS + 1, dtype=torch.float64, device=dev)
    thr = ((RADIUS_MAX * m / RADIUS_BINS) ** 2).to(torch.float32).to(torch.float64)
    lo = torch.zeros(RADIUS_BINS + 2, dtype=torch.int64, device=dev)
    hi = torch.zeros_like(lo)
    k2, p2 = (k * k).sum(1), (p * p).sum(1)
    kq = ((k * 8192.0) == torch.round(k * 8192.0)).all(1)
    pq = ((p * 8192.0) == torch.round(p * 8192.0)).all(1)
    kn, pn = k2.sqrt(), p2.sqrt()
    step = max(1, chunk // max(p.shape[0], 1))
    for a in range(0, k.shape[0], step):
        kk = k[a:a + step]
        d = ((kk[:, None, :] - p[None, :, :]) ** 2).sum(-1)
        e = kc * U24 * (k2[a:a + step, None] + p2[None, :])
        ex = kq[a:a + step, None] & pq[None, :] & ((kn[a:a + step, None] + pn[None, :]) ** 2 < 0.25)
        e = torch.where(ex, torch.zeros_like(e), e)
        # bin b = first m with x < thr_m (RADIUS_BINS + 1: none); cumulative counts follow
        lo += torch.bincount(torch.searchsorted(thr, (d + e).reshape(-1), right=True), minlength=RADIUS_BINS + 2)
        hi += torch.bincount(torch.searchsorted(thr, (d - e).reshape(-1), right=True), minlength=RADIUS_BINS + 2)
    return lo.cumsum(0)[:RADIUS_BINS + 1].cpu().numpy(), hi.cumsum(0)[:RADIUS_BINS + 1].cpu().numpy()


def _pct32(count, denom):
    """points_within_radius.sum().float() / (num_pts * num_kpts) * 100 in fp32 (BUFFERX.py:682-684)."""
    return float(np.float32(np.float32(count) / np.float32(denom)) * np.float32(100.0))


def radius_fp64(lo, hi, denom, threshold, tolerance=0.01):
    """The bisection of BUFFERX.py:675-694 on count intervals [lo[m], hi[m]].  pct is monotone in the count, so a
    decision is decided when the pct of both ends falls on the same side; an undecided one follows every outcome.
    Returns (the set of reachable m, the number of undecided decisions met, the rounded radius of each reachable m)."""
    reach, und = set(), 0
    stack = [(0, RADIUS_BINS, 0)]
    while stack:
        lo_i, hi_i, m = stack.pop()
        if not RADIUS_MAX * hi_i / RADIUS_BINS - RADIUS_MAX * lo_i / RADIUS_BINS > 1e-3:
            reach.add(m)
            continue
        m = (lo_i + hi_i) // 2
        outs = set()
        for c in (lo[m], hi[m]):
            p = _pct32(c, denom)
            outs.add(0 if p < threshold - tolerance else 2 if p > threshold + tolerance else 1)
        if outs == {0, 2}:
            outs.add(1)
        und += len(outs) > 1
        for o in outs:
            if o == 0:
                stack.append((m, hi_i, m))
            elif o == 2:
                stack.append((lo_i, m, m))
            else:
                reach.add(m)
    return reach, und, {mm: np.float32(round(RADIUS_MAX * mm / RADIUS_BINS, 2)) for mm in reach}


def radius_replay(cum, denom, threshold, tolerance=0.01, max_r=5.0):
    """The reference loop literally (BUFFERX.py:674-694) on a cumulative histogram cum[m] = #{d2 < fl32(r_m^2)}: Python
    float64 bisection, torch fp32 percentage, round(des_r, 2).  Returns (m, float32 radius)."""
    low, high, des_r = 0.0, max_r, 0.0
    while high - low > 1e-3:
        des_r = (low + high) / 2.0
        m = int(round(des_r * RADIUS_BINS / max_r))
        assert max_r * m / RADIUS_BINS == des_r
        percentage = (torch.tensor(int(cum[m]), dtype=torch.int64).float() / int(denom) * 100).item()
        if percentage < threshold - tolerance:
            low = des_r
        elif percentage > threshold + tolerance:
            high = des_r
        else:
            break
    return int(round(des_r * RADIUS_BINS / max_r)), np.float32(round(des_r, 2))


def radius_estimation_fp64(src_pts, src_kpts, tgt_pts, tgt_kpts, thresholds, tolerance=0.01, sub_idx=None):
    """density_aware_radius_estimation (BUFFERX.py:627-696) on count intervals: the source only when it has strictly
    more points, pts[sub_idx] above 200000 points with the original N in the denominator.  Returns dict(lo, hi, denom,
    and per threshold (reach, undecided, radii))."""
    if src_pts.shape[0] > tgt_pts.shape[0]:
        pts, kpts = src_pts, src_kpts
    else:
        pts, kpts = tgt_pts, tgt_kpts
    denom = int(pts.shape[0]) * int(kpts.shape[0])
    if pts.shape[0] > 200000:
        pts = pts[sub_idx]
    lo, hi = radius_count_bounds(kpts, pts)
    return dict(lo=lo, hi=hi, denom=denom, per=[radius_fp64(lo, hi, denom, th, tolerance) for th in thresholds])


def ball_query_fp64(xyz, qry, radius, kb=7.0):
    """pointnet2 ``ball_query`` hit test d2 < radius^2 in float64: radius^2 the fp32 product, d64 = sum (q - p)^2.  The
    fp32 d2 = ((dx*dx)+(dy*dy))+(dz*dz), dx = fl(q - p), is within 5u d64 and equals it when every fp32 intermediate is
    exact.  Returns status [Q,N] int8: 1 decided hit, 0 decided miss, 2 undecided ([B,Q,N] for batched xyz [B,N,3],
    qry [B,Q,3])."""
    p, q = _t64(xyz), _t64(qry)
    r = np.float32(radius)
    r2 = float(np.float32(r * r))
    dd = q[..., :, None, :] - p[..., None, :, :]
    sq = dd * dd
    s1 = sq[..., 0] + sq[..., 1]
    d = s1 + sq[..., 2]
    exact = _fits32(dd).all(-1) & _fits32(sq).all(-1) & _fits32(s1) & _fits32(d)
    hit = torch.where(exact, d < r2, d * (1 + kb * U24) < r2)
    miss = torch.where(exact, d >= r2, d * (1 - kb * U24) >= r2)
    st = torch.full(d.shape, 2, dtype=torch.int8, device=d.device)
    st[hit] = 1
    st[miss] = 0
    return st


def select_patches_fp64(pts_perm, kpts, idx):
    """patch_embedder.py:99-111 after the ball query, in float64 on an index row [K,P]: the gathered points, with every
    slot s > 0 whose index equals slot 0's and always slot P-1 replaced by the key point (mask formula)."""
    p, k = _t64(pts_perm), _t64(kpts)
    idx = torch.as_tensor(idx).to(p.device).long()
    P = idx.shape[1]
    new_points = p[idx]
    mask = (idx == idx[:, :1].repeat(1, P)).to(torch.float64)
    mask[:, 0] = 0
    mask[:, P - 1] = 1
    mask = mask.unsqueeze(2)
    return new_points * (1 - mask) + k.unsqueeze(1) * mask


# --------------------------------------------------------------------------- #
# a10, a13-a15 evaluated in float64 from the reference's formulas (tests/test_pose_fp64_*.py)
# --------------------------------------------------------------------------- #
def mutual_nn_fp64(a, b):
    """knn_cuda KNN(k=1) both ways on the fp32 descriptors, distances sum (a - b)^2 in float64 -> dict(D [Ka,Kb], and per
    row (r_*) and per column (c_*): the best and second-best distance and the best's index (first minimum))."""
    a = np.asarray(a, np.float32).astype(np.float64)
    b = np.asarray(b, np.float32).astype(np.float64)
    D = ((a[:, None, :] - b[None, :, :]) ** 2).sum(-1) if a.size and b.size else np.zeros((len(a), len(b)))
    out = dict(D=D)
    for side, M in (("r", D), ("c", D.T)):
        n = M.shape[1]
        srt = np.sort(M, axis=1) if n else np.zeros((M.shape[0], 0))
        out[side + "_idx"] = M.argmin(1) if n else np.zeros(M.shape[0], np.int64)
        out[side + "_best"] = srt[:, 0] if n else np.full(M.shape[0], np.inf)
        out[side + "_second"] = srt[:, 1] if n > 1 else np.full(M.shape[0], np.inf)
    return out


def consensus_fp64(ss, tt, R, t, azi_n, inlier_th):
    """BUFFERX.py:404-417 literally, in float64 on the fp32 inputs: diffs [Mc,Mc] (hypothesis j, correspondence i),
    thr [Mc], sign = diffs < thr, counts, best = first arg-max."""
    ss, tt, R, t = (torch.from_numpy(np.asarray(x, np.float32).astype(np.float64)) for x in (ss, tt, R, t))
    tss = ss[None] @ R.transpose(-1, -2) + t[:, None]
    diffs = torch.sqrt(torch.sum((tss - tt[None]) ** 2, dim=-1))
    thr = torch.sqrt(torch.sum(ss ** 2, dim=-1)) * np.pi / azi_n * float(np.float32(inlier_th))
    sign = diffs < thr[None]
    counts = torch.sum(sign, dim=-1)
    best = int(torch.argmax(counts)) if len(counts) else 0
    return dict(diffs=diffs.numpy(), thr=thr.numpy(), sign=sign.numpy(), counts=counts.numpy(), best=best)


def umeyama_fp64(a, b, w=None):
    """Rigid fit without scale (Umeyama / Open3D TransformationEstimationPointToPoint(False)) in float64: weighted
    centroids, H = sum w (a - ca)(b - cb)^T, H = U S V^T, d = sign det(V U^T), R = V diag(1, 1, d) U^T, t = cb - R ca.
    -> dict(R, t, ca, cb, sv (singular values, descending), d)."""
    a = np.asarray(a, np.float64).reshape(-1, 3)
    b = np.asarray(b, np.float64).reshape(-1, 3)
    w = np.ones(len(a)) if w is None else np.asarray(w, np.float64)
    sw = w.sum()
    ca, cb = (w[:, None] * a).sum(0) / sw, (w[:, None] * b).sum(0) / sw
    H = (w[:, None] * (a - ca)).T @ (b - cb)
    U, S, Vt = np.linalg.svd(H)
    d = 1.0 if np.linalg.det(Vt.T @ U.T) >= 0 else -1.0
    R = Vt.T @ np.diag([1.0, 1.0, d]) @ U.T
    return dict(R=R, t=cb - R @ ca, ca=ca, cb=cb, sv=S, d=d)


def philox4x32_10_np(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11) in NumPy: ctr [n,4] / key [2] uint32 -> [n,4] uint32."""
    c = [np.asarray(ctr, np.uint64)[:, i].copy() for i in range(4)]
    k0, k1 = np.uint64(int(key[0]) & 0xFFFFFFFF), np.uint64(int(key[1]) & 0xFFFFFFFF)
    m32 = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & m32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & m32]
        k0 = (k0 + np.uint64(0x9E3779B9)) & m32
        k1 = (k1 + np.uint64(0xBB67AE85)) & m32
    return np.stack(c, axis=1).astype(np.uint32)


def ransac_draws(seed, I, n):
    """The three correspondence draws of iterations 0..n-1: counter (itr, 0, 0, 0), key (seed lo, seed hi),
    sel = (rnd * I) >> 32 -> [n,3] int64."""
    ctr = np.zeros((n, 4), np.uint64)
    ctr[:, 0] = np.arange(n, dtype=np.uint64)
    rnd = philox4x32_10_np(ctr, (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF))[:, :3].astype(np.uint64)
    return ((rnd * np.uint64(I)) >> np.uint64(32)).astype(np.int64)


def refine_fp64(src, tgt, T_in, dist_th):
    """post_refinement + rigid_transform_3d (BUFFERX.py:522-603) literally, in torch float64 on the fp32 inputs: 20 rounds
    at dist_th, stop when |inliers - previous| < 1, weights 1 / (1 + (d / th)^2), centroids over (sum w + 1e-6), torch.svd
    and the det correction.  -> dict(T (final), rounds, per round: T used, d [n], mask, and the fit's (w, R, t))."""
    src = torch.from_numpy(np.asarray(src, np.float32).astype(np.float64))[None]
    tgt = torch.from_numpy(np.asarray(tgt, np.float32).astype(np.float64))[None]
    tr = torch.from_numpy(np.asarray(T_in, np.float32).astype(np.float64).reshape(4, 4))[None]
    th = float(np.float32(dist_th))
    prev, hist, r = 0, [], 0
    while r < 20:
        L2 =torch.norm((tr[:, :3, :3] @ src.permute(0, 2, 1) + tr[:, :3, 3:4]).permute(0, 2, 1) - tgt, dim=-1)
        pred = (L2 < th)[0]
        n = int(pred.sum())
        step = dict(T=tr[0].numpy().copy(), d=L2[0].numpy().copy(), mask=pred.numpy().copy())
        hist.append(step)
        if abs(n - prev) < 1:
            break
        prev = n
        A, B, wt = src[:, pred], tgt[:, pred], (1 / (1 + (L2 / th) ** 2))[:, pred]
        cA = (A * wt[:, :, None]).sum(1, keepdim=True) / (wt.sum(1, keepdim=True)[:, :, None] + 1e-6)
        cB = (B * wt[:, :, None]).sum(1, keepdim=True) / (wt.sum(1, keepdim=True)[:, :, None] + 1e-6)
        H = (A - cA).permute(0, 2, 1) @ torch.diag_embed(wt) @ (B - cB)
        U, S, V = torch.svd(H)
        eye = torch.eye(3, dtype=torch.float64)[None].clone()
        eye[:, -1, -1] = torch.det(V @ U.permute(0, 2, 1))
        R = V @ eye @ U.permute(0, 2, 1)
        tr = torch.eye(4, dtype=torch.float64)[None].clone()
        tr[:, :3, :3], tr[:, :3, 3:4] = R, cB.permute(0, 2, 1) - R @ cA.permute(0, 2, 1)
        step.update(w=wt[0].numpy().copy(), R=R[0].numpy().copy(), t=tr[0, :3, 3].numpy().copy(), sv=S[0].numpy().copy(),
                    cA=cA[0, 0].numpy().copy(), cB=cB[0, 0].numpy().copy())
        r += 1
    return dict(T=tr[0].numpy().copy(), rounds=r, hist=hist)


U53 = 2.0 ** -53


def fit_bounds(a, b, kf=16.0):
    """Umeyama on one triple (or any set) and what bounds a float64 fit of it: bR (largest entry of R - R64, from
    |dH| <= kf u53 sum |a - ca| |b - cb| over the gap sigma_2 + d sigma_3), or inf when the fit is degenerate (bR > 1e-6:
    duplicate, collinear or coincident points, where the rotation about the line is free); the line (unit u through ca,
    v through cb) and the largest off-line distance of the points for that case."""
    f = umeyama_fp64(a, b)
    a = np.asarray(a, np.float64).reshape(-1, 3)
    b = np.asarray(b, np.float64).reshape(-1, 3)
    da, db = a - f["ca"], b - f["cb"]
    dH = kf * U53 * (np.linalg.norm(da, axis=1) * np.linalg.norm(db, axis=1)).sum()
    gap = f["sv"][1] + f["d"] * f["sv"][2]
    bR = 2.0 * dH / gap if gap > 0 else np.inf
    f["bR"] = bR if bR <= 1e-6 else np.inf
    U, _, Vt = np.linalg.svd(da.T @ db)
    u, v = U[:, 0], Vt[0]
    f["line"] = (u, v, f["sv"][0] > 0)
    f["off"] = max(np.linalg.norm(da - np.outer(da @ u, u), axis=1).max(), np.linalg.norm(db - np.outer(db @ v, v), axis=1).max())
    return f


def _fit_dist(f, x, g, kf=16.0):
    """|T64 x - g| and its margin for a fit of bound f["bR"]: a rotation error bR per entry moves x by <= 3 bR |x - ca|,
    plus kf u53 of the magnitudes (centroids, evaluation)."""
    x, g = np.asarray(x, np.float64).reshape(-1, 3), np.asarray(g, np.float64).reshape(-1, 3)
    e = np.linalg.norm(x @ f["R"].T + f["t"] - g, axis=1)
    m = 3 * f["bR"] * np.linalg.norm(x - f["ca"], axis=1) + kf * U53 * (np.abs(f["ca"]).sum() + np.abs(f["cb"]).sum()
                                                                        + 3 * np.abs(x).sum(1) + np.abs(g).sum(1) + e)
    return e, m


def _line_dist(f, x, g):
    """Smallest |T x - g| over every rigid T that maps the fit's line onto its target line and ca onto cb (the free
    rotation of a degenerate triple): the cylinder coordinates (h, rho) of x about (ca, u) and of g about (cb, v); for a
    coincident triple (no line), | |x - ca| - |g - cb| |."""
    x, g = np.asarray(x, np.float64).reshape(-1, 3), np.asarray(g, np.float64).reshape(-1, 3)
    u, v, has_line = f["line"]
    dx, dg = x - f["ca"], g - f["cb"]
    if not has_line:
        return np.abs(np.linalg.norm(dx, axis=1) - np.linalg.norm(dg, axis=1))
    hx, hg = dx @ u, dg @ v
    rx, rg = np.linalg.norm(dx - np.outer(hx, u), axis=1), np.linalg.norm(dg - np.outer(hg, v), axis=1)
    return np.hypot(hx - hg, rx - rg)


def ransac_fp64(src, tgt, inlier_ind, dist_th, similar_th, confidence, max_iter, seed, ke=8.0, kf=16.0, recs=None):
    """RegistrationRANSACBasedOnCorrespondence replayed in float64 on the kernel's draws (``ransac_draws``): per
    iteration the EdgeLength checker, the Umeyama fit of the triple, the Distance checker, the inlier count and rmse; then
    Open3D's sequential bookkeeping (more inliers wins, then lower rmse; est_k = ceil(log(1 - conf) / log(1 - r^3))).
    Every decision within its rounding margin is flagged: the checkers (ke u53 of the edge lengths; the fit margin of
    ``_fit_dist``), each inlier test (-> a count interval [lo, hi]), the rmse tie-break and est_k near an integer.  A
    degenerate triple (``fit_bounds``) has a free rotation about its line: its Distance checker is decided only for
    points on that line and its count lies in [0, hi] with hi from ``_line_dist``; it cannot win once hi < best.  With
    ``recs`` (an implementation's per-iteration records) a degenerate iteration takes the recorded count and rmse -- its
    own choice among the equally good rotations -- once that count is shown to lie in [0, hi].
    -> dict(num_inliers, best_itr, iters, first_marginal (itr or None), recs (per iteration), fits (itr -> fit))."""
    S = np.asarray(src, np.float32).astype(np.float64)
    D = np.asarray(tgt, np.float32).astype(np.float64)
    ind = np.asarray(inlier_ind, np.int64)
    I = len(ind)
    out = dict(num_inliers=0, best_itr=-1, iters=0, first_marginal=None, recs=[], fits={})
    if I < 3 or max_iter <= 0:
        return out
    s, g = S[ind], D[ind]
    sel_all = ransac_draws(seed, I, max_iter)
    th = float(dist_th)
    best_good, best_rmse, best_itr, best_sel, best_dr, est_k = 0, 0.0, -1, None, 0.0, max_iter
    first_marg = None

    def marg(itr):
        nonlocal first_marg
        if first_marg is None:
            first_marg = itr

    itr = 0
    while itr < max_iter and itr < est_k:
        sel = sel_all[itr]
        a, b = s[sel], g[sel]
        rec = dict(itr=itr, sel=tuple(sel), passed=False, marginal=False, deg=False, lo=0, hi=0, rmse=0.0)
        out["recs"].append(rec)
        ok = True
        for i in range(3):
            for j in range(i + 1, 3):
                ds, dt = np.linalg.norm(a[i] - a[j]), np.linalg.norm(b[i] - b[j])
                m = ke * U53 * (ds + dt)
                if abs(ds - dt * similar_th) < m or abs(dt - ds * similar_th) < m:
                    rec["marginal"] = True
                if ds < dt * similar_th or dt < ds * similar_th:
                    ok = False
        if ok:
            f = fit_bounds(a, b, kf)
            out["fits"][itr] = f
            rec["deg"] = deg = not np.isfinite(f["bR"])
            if deg:
                e = np.linalg.norm(a @ f["R"].T + f["t"] - b, axis=1)
                m = 2 * f["off"] + kf * U53 * (np.abs(a).sum(1) + np.abs(b).sum(1) + 1)
            else:
                e, m = _fit_dist(f, a, b, kf)
            if (np.abs(e - th) <= m).any():
                rec["marginal"] = True
            ok = not (e > th).any()
        rec["passed"] = ok
        if rec["marginal"]:
            marg(itr)
        if not ok:
            itr += 1
            continue
        if deg:
            ld = _line_dist(f, s, g)
            rec["hi"] = hi = int((ld < th + 2 * f["off"] + kf * U53 * (np.abs(s).sum(1) + np.abs(g).sum(1))).sum())
            if recs is not None and itr < len(recs) and recs["pass"][itr]:
                good, rmse, dr = int(recs["good"][itr]), float(recs["rmse"][itr]), 0.0
                assert good <= hi, f"itr {itr}: a degenerate triple counted {good} inliers, more than the {hi} its line allows"
                rec["lo"] = rec["hi"] = good
                rec["rmse"] = rmse
            else:
                if not (hi < best_good or (hi == 0 and best_good == 0)):
                    marg(itr)
                    rec["marginal"] = True
                itr += 1
                continue
        else:
            e, m = _fit_dist(f, s, g, kf)
            inl = e < th
            mg = np.abs(e - th) <= m
            rec["lo"], rec["hi"] = lo, hi = int((inl & ~mg).sum()), int((inl | mg).sum())
            good = int(inl.sum())
            rmse = float(np.sqrt((e[inl] ** 2).sum() / good)) if good else 0.0
            dr = float(m.max()) if good else 0.0
            rec["rmse"] = rmse
            if lo != hi and hi >= best_good:
                marg(itr)
                rec["marginal"] = True
        better = good > best_good or (good == best_good and rmse < best_rmse)
        if good == best_good and good > 0 and tuple(sel) != best_sel and abs(rmse - best_rmse) <= dr + best_dr:
            marg(itr)
            rec["marginal"] = True
        if better:
            best_good, best_rmse, best_itr, best_sel, best_dr = good, rmse, itr, tuple(sel), dr
            with np.errstate(divide="ignore", invalid="ignore"):
                est = float(np.log(np.float64(1.0 - confidence)) / np.log(np.float64(1.0 - (good / I) ** 3)))
            if np.isfinite(est) and abs(est - round(est)) <= 1e-9 * abs(est) and est != 0:
                marg(itr)
            if est < est_k:
                est_k = int(math.ceil(est))
        itr += 1
    out.update(num_inliers=best_good, best_itr=best_itr, iters=itr, first_marginal=first_marg)
    return out


# --------------------------------------------------------------------------- #
# conv stacks (torch CPU fp32) -- functional over a reference-keyed state_dict
# --------------------------------------------------------------------------- #
def _bn(x, sd, pfx, affine):
    w = sd[pfx + ".weight"] if affine else None
    b = sd[pfx + ".bias"] if affine else None
    return F.batch_norm(x, sd[pfx + ".running_mean"], sd[pfx + ".running_var"], w, b, training=False, eps=1e-5)


def _pad_cyl(x):
    """Circular +-1 along the last (azimuth) axis, zero +-1 along the second-last (elevation) axis
    (``utils/common.py:265-310`` for kernel size 3); any leading axes are left alone."""
    x = torch.cat([x[..., -1:], x, x[..., :1]], dim=-1)
    pad = [0, 0, 1, 1]  # (last: none, second-last: 1 each side)
    return F.pad(x, pad)


def pnt_max(inv_patches: torch.Tensor, sd, pfx="Desc.") -> torch.Tensor:
    """a7: [K,V,nv,3] -> [K,16,V] (1x1 conv + BN + ReLU per sample, max over the nv samples)."""
    x = inv_patches.permute(0, 3, 1, 2)
    x = F.conv2d(x, sd[pfx + "pnt_layer.0.weight"], sd[pfx + "pnt_layer.0.bias"])
    x = F.relu(_bn(x, sd, pfx + "pnt_layer.1", True))
    return x.max(dim=3).values


_CYL_CONVS = [0, 3, 6, 9, 12, 15, 18, 21]


def _cyl_layers(x: torch.Tensor, sd, pfx, keep=False):
    """The eight Cylindrical_Net layers in the dtype of x and ``sd`` -> (output [K,32,7,20], the activation after each
    layer if ``keep``: post-ReLU for the first seven, the plain convolution for the last)."""
    x = F.conv3d(_pad_cyl(x), sd[pfx + "ops.0.weight"], sd[pfx + "ops.0.bias"])
    x = F.relu(_bn(x, sd, pfx + "ops.1", False)).squeeze(2)
    acts = [x] if keep else []
    for i in _CYL_CONVS[1:]:
        x = F.conv2d(_pad_cyl(x), sd[pfx + f"ops.{i}.weight"], sd[pfx + f"ops.{i}.bias"])
        if i != 21:
            x = F.relu(_bn(x, sd, pfx + f"ops.{i + 1}", False))
        if keep:
            acts.append(x)
    return x, acts


def cyl_net(x: torch.Tensor, sd, pfx="Desc.conv_net.") -> torch.Tensor:
    """a8: [K,16,3,7,20] -> [K,32,7,20]."""
    return _cyl_layers(x, sd, pfx)[0]


def _pool(x: torch.Tensor, sd, pfx):
    """a9 -> (desc [K,32], equi [K,32,7,20], attention map [K,1,7,20], pooled vector before the normalisation [K,32])."""
    w = F.conv2d(x, sd[pfx + "pool_layer.0.weight"], sd[pfx + "pool_layer.0.bias"])
    w = F.relu(_bn(w, sd, pfx + "pool_layer.1", True))
    w = F.conv2d(w, sd[pfx + "pool_layer.3.weight"], sd[pfx + "pool_layer.3.bias"])
    w = F.relu(_bn(w, sd, pfx + "pool_layer.4", True))
    f = F.avg_pool2d(x * w, kernel_size=(x.shape[2], x.shape[3])).view(x.shape[0], -1)
    return F.normalize(f, p=2, dim=1), F.normalize(x, p=2, dim=1), w, f


def pool_desc(x: torch.Tensor, sd, pfx="Desc."):
    """a9: x [K,32,7,20] -> desc [K,32] (L2-normalised attention-pooled), equi [K,32,7,20]."""
    d, e, _, _ = _pool(x, sd, pfx)
    return d, e


def _sd64(sd, pfx, device):
    return {k: (v.double() if v.is_floating_point() else v).to(device) for k, v in sd.items() if k.startswith(pfx)}


def desc_fp64(feat: torch.Tensor, sd, keep=False, rad_n=3, ele_n=7, azi_n=20):
    """a8+a9 evaluated in float64 on the point-layer features [k,16,V] (on their device: torch's own float64 kernels): the
    ground truth against which the fp32 oracle and the GPU path are both measured (tests/test_gpu_parity.py,
    tests/test_descnet_fp64_*.py).  -> desc [k,32] float64; with ``keep`` also a dict: ``acts`` (the eight layer outputs of
    _cyl_layers), ``equi``, ``att`` (attention map [k,1,7,20]) and ``pooled`` (the vector before its L2 normalisation)."""
    sd64 = _sd64(sd, "Desc.", feat.device)
    with torch.no_grad():
        x, acts = _cyl_layers(feat.double().view(feat.shape[0], feat.shape[1], rad_n, ele_n, azi_n), sd64, "Desc.conv_net.", keep)
        d, equi, att, pooled = _pool(x, sd64, "Desc.")
    return (d, dict(acts=acts, equi=equi, att=att, pooled=pooled)) if keep else d


def pnt_fp64(delta, vidx, sd, absref=False, azi_n=20, pfx="Desc."):
    """a7 in float64 on an integer voxel selection: delta [K,P,3] fp32 patches, vidx [K,V,nv] (oracle.spt's) -> the
    point-layer features [K,16,V] float64.  The samples are de-rotated in float64 (angle -a 2 pi / azi_n) from the fp32
    coordinates; a slot is zero where oracle.spt zeroes it (slot 0 holding index 0, padding slots repeating slot 0).  With
    ``absref`` also max over the samples of |W| |x'| + |b| (conv + BN folded in float64; |x'| from |x| |cos| + |y| |sin|, so
    that a cancelling de-rotation does not shrink the bound), on the same device as the features."""
    delta = torch.as_tensor(np.asarray(delta) if not isinstance(delta, torch.Tensor) else delta)
    vidx = torch.as_tensor(np.asarray(vidx) if not isinstance(vidx, torch.Tensor) else vidx).long().to(delta.device)
    K, V, nv = vidx.shape
    dev = delta.device
    d = delta.double()
    pts = torch.gather(d, 1, vidx.view(K, V * nv, 1).expand(K, V * nv, 3)).view(K, V, nv, 3)
    zero = torch.zeros((K, V, nv), dtype=torch.bool, device=dev)
    zero[:, :, 0] = vidx[:, :, 0] == 0
    zero[:, :, 1:] = vidx[:, :, 1:] == vidx[:, :, :1]
    pts = torch.where(zero[..., None], torch.zeros((), dtype=torch.float64, device=dev), pts)
    ang = -torch.arange(azi_n, dtype=torch.float64, device=dev) * (2 * math.pi / azi_n)
    a = torch.arange(V, device=dev) % azi_n
    c, s = torch.cos(ang)[a].view(1, V, 1), torch.sin(ang)[a].view(1, V, 1)
    x, y, z = pts[..., 0], pts[..., 1], pts[..., 2]
    inv = torch.stack([x * c - y * s, x * s + y * c, z], dim=-1)                  # [K,V,nv,3]
    g = lambda k: sd[pfx + k].detach().double().to(dev)
    sc = g("pnt_layer.1.weight") / torch.sqrt(g("pnt_layer.1.running_var") + 1e-5)
    W = g("pnt_layer.0.weight").view(16, 3) * sc[:, None]
    b = (g("pnt_layer.0.bias") - g("pnt_layer.1.running_mean")) * sc + g("pnt_layer.1.bias")
    feat = torch.relu(inv @ W.t() + b).amax(dim=2).permute(0, 2, 1).contiguous()
    if not absref:
        return feat
    ax = torch.stack([x.abs() * c.abs() + y.abs() * s.abs(), x.abs() * s.abs() + y.abs() * c.abs(), z.abs()], dim=-1)
    return feat, (ax @ W.abs().t() + b.abs()).amax(dim=2).permute(0, 2, 1).contiguous()


_COST_CONVS = [0, 3, 6, 9, 12, 15, 18, 21, 24, 27]


def _cost_net(d1: torch.Tensor, d2: torch.Tensor, sd, azi_n, pfx, keep=False):
    """The cost volume of d1,d2 [M,32,5,20] through CostNet in the dtype of the inputs and ``sd`` -> (logits [M,azi_n],
    post-ReLU activations of the nine hidden layers if ``keep``)."""
    M = d1.shape[0]
    l = torch.arange(azi_n)
    idx = (l[None, :] - l[:, None]) % azi_n          # idx[n][l] = (l - n) mod azi_n  (BUFFERX.py:43-48)
    x = d1[:, :, :, idx.reshape(-1)].reshape(M, d1.shape[1], d1.shape[2], azi_n, azi_n)
    x = x.permute(0, 1, 3, 2, 4) - d2.unsqueeze(2)   # [M,C,n,k,l]
    acts = []
    for i in _COST_CONVS:
        x = F.conv3d(x, sd[pfx + f"ops.{i}.weight"], sd[pfx + f"ops.{i}.bias"])
        if i != 27:
            x = F.relu(_bn(x, sd, pfx + f"ops.{i + 1}", False))
            if keep:
                acts.append(x)
    return x.reshape(M, azi_n), acts


def cost_volume(d1: torch.Tensor, d2: torch.Tensor, sd, azi_n=20, pfx="Pose.conv.") -> torch.Tensor:
    """a11: d1,d2 [M,32,5,20] -> soft arg-max azimuth bin [M] (float)."""
    M = d1.shape[0]
    if M == 0:
        return torch.zeros(0)
    cost, _ = _cost_net(d1, d2, sd, azi_n, pfx)
    prob = F.softmax(cost, dim=-1)
    return torch.sum(prob * torch.arange(0, azi_n)[None], dim=-1)


def costnet_fp64(d1: torch.Tensor, d2: torch.Tensor, sd, keep=False, azi_n=20, pfx="Pose.conv."):
    """a11 evaluated in float64 on the (fp32) maps d1,d2 [M,32,5,20] -> logits [M,azi_n] float64; with ``keep`` also the
    post-ReLU activation of every hidden layer.  The ground truth against which the fp32 oracle and every CostNet kernel
    are measured (tests/test_costnet_fp64_*.py)."""
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items() if k.startswith(pfx)}
    with torch.no_grad():
        logits, acts = _cost_net(d1.double(), d2.double(), sd64, azi_n, pfx, keep)
    return (logits, acts) if keep else logits


def soft_argmax(logits: torch.Tensor) -> torch.Tensor:
    """The reference's non-circular expectation sum(softmax(logits) * arange) (BUFFERX.py:66-69), in float64."""
    lg = torch.as_tensor(logits).double()
    prob = F.softmax(lg, dim=-1)
    return torch.sum(prob * torch.arange(lg.shape[-1], dtype=torch.float64)[None], dim=-1)


def soft_argmax_bound(l64: torch.Tensor, l32: torch.Tensor):
    """The a11 bound on a soft arg-max bin against float64 logits ``l64``, given the fp32 oracle's logits ``l32`` of the same
    rows -> (ind64, bound, s, ind32_err).  1e-4 (about 10x the fp32 oracle's error on a single peak), scaled by
    s = sum p_k |k - ind| (d ind / d logit_k = p_k (k - ind), so a row whose mass sits at both ends of the bin range turns
    the same fp32-grade logit error into a larger bin error; s <= 1 on a single peak), at least 1.5 x the fp32 oracle's own
    error on the row, never beyond 2e-4."""
    ind64 = soft_argmax(l64)
    ind32_err = (soft_argmax(l32) - ind64).abs()
    p = torch.softmax(l64, dim=1)
    s = (p * (torch.arange(l64.shape[1], dtype=torch.float64)[None] - ind64[:, None]).abs()).sum(dim=1)
    bound = torch.clamp(torch.maximum(1e-4 * s.clamp(min=1.0), 1.5 * ind32_err), max=2e-4)
    return ind64, bound, s, ind32_err


def azimuth_rotation(angle: torch.Tensor, _mutations=()) -> torch.Tensor:
    """kornia ``axis_angle_to_rotation_matrix`` for the axis-angle (0,0,angle) (BUFFERX.py:383-386).  ``_mutations``
    (tests/test_train_fp64_cpu.py only): "no_eps" drops the + 1e-6 of the axis, "ge_threshold" takes the full form at
    theta^2 >= 1e-6."""
    theta2 = angle * angle
    theta = torch.sqrt(theta2)
    wz = angle / theta if "no_eps" in _mutations else angle / (theta + 1e-6)
    c, s = torch.cos(theta), torch.sin(theta)
    one, zero = torch.ones_like(c), torch.zeros_like(c)
    Rn = torch.stack([c, -wz * s, zero, wz * s, c, zero, zero, zero, c + wz * wz * (one - c)], dim=1).view(-1, 3, 3)
    Rt = torch.stack([one, -angle, zero, angle, one, zero, zero, zero, one], dim=1).view(-1, 3, 3)
    mask = ((theta2 >= 1e-6) if "ge_threshold" in _mutations else (theta2 > 1e-6)).view(-1, 1, 1)
    return torch.where(mask, Rn, Rt)


def hypotheses(ind, ss_kpts, tt_kpts, ss_R, tt_R, azi_n=20):
    """a12 (BUFFERX.py:382-389): R = tt_R @ Rz(angle) @ ss_R^T, t = tt_kpt - R ss_kpt."""
    angle = ind * 2 * np.pi / azi_n + 1e-6
    azi_R = azimuth_rotation(angle)
    R = tt_R @ azi_R @ ss_R.transpose(-1, -2)
    t = tt_kpts - (R @ ss_kpts.unsqueeze(-1)).squeeze(-1)
    return R, t


# --------------------------------------------------------------------------- #
# descriptor + full pair
# --------------------------------------------------------------------------- #
def describe(sd, cfg, pts, kpts, des_r: float, aligned: bool, perm, keep=False, timings=None, z_axis=None):
    """MiniSpinNet.forward in eval mode (patch_embedder.py:44-90) for one cloud."""
    P = cfg.patch.num_points_per_patch
    rad_n, azi_n, ele_n = cfg.patch.rad_n, cfg.patch.azi_n, cfg.patch.ele_n
    t0 = time.perf_counter()
    idx, patches = select_patches(pts, perm, kpts, des_r, P)
    t1 = time.perf_counter()
    delta, Rt, rand_axis, z_used = lrf(patches, des_r, aligned, z_axis=z_axis, want_z=True)
    t2 = time.perf_counter()
    inv, vidx = spt(delta, rad_n, azi_n, ele_n, cfg.patch.delta / rad_n, cfg.patch.voxel_sample)
    t3 = time.perf_counter()
    with torch.no_grad():
        feat = pnt_max(torch.from_numpy(inv), sd)
        x = cyl_net(feat.view(feat.shape[0], feat.shape[1], rad_n, ele_n, azi_n), sd)
        desc, equi = pool_desc(x, sd)
    t4 = time.perf_counter()
    if timings is not None:
        for k, v in (("ball_query_group", t1 - t0), ("lrf", t2 - t1), ("spt", t3 - t2), ("conv_desc", t4 - t3)):
            timings[k] = timings.get(k, 0.0) + v
    out = dict(desc=desc, equi=equi, R=torch.from_numpy(Rt), rand_axis=torch.from_numpy(rand_axis))
    if keep:
        out.update(idx=idx, patches=patches, delta=delta, inv=inv, vidx=vidx, feat=feat, x=x, z=z_used)
    return out


def draw_perms(cfg, n_src, n_tgt, seed):
    """The host permutations the reference draws from NumPy's global RNG (patch_embedder.py:96),
    src then tgt per scale, made explicit: ``np.random.seed(seed)`` + the same calls."""
    st = np.random.RandomState(seed)
    perms = []
    for _ in range(cfg.patch.num_scales):
        perms.append((st.choice(n_src, n_src, replace=False).astype(np.int32),
                      st.choice(n_tgt, n_tgt, replace=False).astype(np.int32)))
    return perms


def should_exit(cfg, num_inliers):
    """``PoseEstimator.compute_confidence_score`` (pose_estimator.py:119-126)."""
    return num_inliers >= cfg.match.get("early_exit_min_inliers", 15)


def register_pair(sd, cfg, data, perms, ransac_seed=0, keep=False, timings=None, z_axes=None, sub_idx=None):
    """``BufferX.forward`` inference branch (models/BUFFERX.py:257-467), early exit disabled or enabled
    as configured.  Returns (pose, num_inliers, num_mutual, num_inlier_ind, scales_used, aux).
    ``z_axes`` (ref_check.py only): per scale a (src [K,3], tgt [K,3]) pair of LRF z axes to impose.
    A larger cloud of more than 200000 points is sub-sampled once per scale that runs, as the reference does
    (BUFFERX.py:320-329 calls the radius estimation inside the scale loop): scale i histograms ``sub_idx[i]``, or without
    ``sub_idx`` its own draw from torch's CPU generator, made in scale order (one draw after an early exit at scale 0)."""
    src = _f32(data["src_fds_pcd"])
    tgt = _f32(data["tgt_fds_pcd"])
    aligned = bool(data["is_aligned_to_global_z"])
    Kr = cfg.patch.num_points_radius_estimate
    K = cfg.patch.num_fps
    azi_n = cfg.patch.azi_n
    tm = timings if timings is not None else {}

    def _t(name, t0):
        tm[name] = tm.get(name, 0.0) + (time.perf_counter() - t0)

    t0 = time.perf_counter()
    s_idx_r = fps(src, Kr)
    t_idx_r = fps(tgt, Kr)
    # the per-scale FPS(num_fps) calls of the reference are deterministic repeats (BUFFERX.py:338-339)
    s_idx = s_idx_r[:K] if K <= Kr else fps(src, K)
    t_idx = t_idx_r[:K] if K <= Kr else fps(tgt, K)
    _t("fps", t0)
    kpts1, kpts2 = src[s_idx_r], tgt[t_idx_r]
    src_kpts, tgt_kpts = src[s_idx], tgt[t_idx]

    t0 = time.perf_counter()
    cum = None                      # up to 200000 points one histogram serves every scale
    if max(src.shape[0], tgt.shape[0]) <= 200000:
        cum = radius_hist(kpts1, src) if src.shape[0] > tgt.shape[0] else radius_hist(kpts2, tgt)
    _t("radius_estimation", t0)

    enable_early_exit = cfg.match.get("enable_early_exit", True)
    aux = dict(des_r=[], scales=[], s_fps=s_idx_r, t_fps=t_idx_r, ransac_calls=[])
    R_acc, t_acc, ss_acc, tt_acc = [], [], [], []
    init_pose, num_inliers, scales_used, exit_now = None, 0, 0, False
    inlier_ind = np.zeros(0, dtype=np.int32)
    for i in range(cfg.patch.num_scales):
        t0 = time.perf_counter()
        th = [cfg.patch.search_radius_thresholds[i]]
        if sub_idx is None:
            des_r = radius_estimation(src, kpts1, tgt, kpts2, th, cum=cum)[0]
        else:
            des_r = radius_estimation(src, kpts1, tgt, kpts2, th, cum=cum, sub_idx=sub_idx[i])[0]
        _t("radius_estimation", t0)
        aux["des_r"].append(des_r)
        zs, zt = (None, None) if z_axes is None else z_axes[i]
        s = describe(sd, cfg, src, src_kpts, des_r, aligned, perms[i][0], keep=keep, timings=tm, z_axis=zs)
        t = describe(sd, cfg, tgt, tgt_kpts, des_r, aligned, perms[i][1], keep=keep, timings=tm, z_axis=zt)
        t0 = time.perf_counter()
        s_m, t_m, snn, tnn = mutual_nn(s["desc"].numpy(), t["desc"].numpy())
        _t("mutual_nn", t0)
        sm, tm_ = torch.from_numpy(s_m.astype(np.int64)), torch.from_numpy(t_m.astype(np.int64))
        ss_kpts, tt_kpts = torch.from_numpy(src_kpts)[sm], torch.from_numpy(tgt_kpts)[tm_]
        t0 = time.perf_counter()
        with torch.no_grad():
            ind = cost_volume(s["equi"][sm][:, :, 1:cfg.patch.ele_n - 1], t["equi"][tm_][:, :, 1:cfg.patch.ele_n - 1], sd, azi_n)
            R, tr = hypotheses(ind, ss_kpts, tt_kpts, s["R"][sm], t["R"][tm_], azi_n)
        _t("cost_volume", t0)
        R_acc.append(R); t_acc.append(tr); ss_acc.append(ss_kpts); tt_acc.append(tt_kpts)
        scales_used = i + 1
        R_cat, t_cat = torch.cat(R_acc), torch.cat(t_acc)
        ss_cat, tt_cat = torch.cat(ss_acc), torch.cat(tt_acc)
        t0 = time.perf_counter()
        inlier_ind, best, counts = consensus(ss_cat.numpy(), tt_cat.numpy(), R_cat.numpy(), t_cat.numpy(), azi_n,
                                             cfg.match.inlier_th)
        _t("consensus", t0)
        sc = dict(s_mids=s_m, t_mids=t_m, ind=ind.numpy(), R=R.numpy(), t=tr.numpy(), best=best, counts=counts,
                  inlier_ind=inlier_ind, snn=snn, tnn=tnn, src=s, tgt=t)
        aux["scales"].append(sc)
        if enable_early_exit and i == 0:
            t0 = time.perf_counter()
            r = ransac(ss_cat.numpy(), tt_cat.numpy(), inlier_ind, cfg.match.dist_th, cfg.match.similar_th,
                       cfg.match.confidence, cfg.match.iter_n, ransac_seed)
            _t("ransac", t0)
            aux["ransac_calls"].append(dict(inlier_ind=inlier_ind.copy(), **r))
            init_pose, num_inliers = r["T"], r["num_inliers"]
            exit_now = should_exit(cfg, num_inliers)
            if exit_now:
                break
    num_mutual = int(ss_cat.shape[0])
    if (not enable_early_exit) or (enable_early_exit and not exit_now):
        t0 = time.perf_counter()
        r = ransac(ss_cat.numpy(), tt_cat.numpy(), inlier_ind, cfg.match.dist_th, cfg.match.similar_th,
                   cfg.match.confidence, cfg.match.iter_n, ransac_seed)
        _t("ransac", t0)
        aux["ransac_calls"].append(dict(inlier_ind=inlier_ind.copy(), **r))
        init_pose, num_inliers = r["T"], r["num_inliers"]
        aux["ransac"] = r
    aux["init_pose"] = init_pose
    if cfg.test.pose_refine is True:
        t0 = time.perf_counter()
        pose, rounds = refine(ss_cat.numpy(), tt_cat.numpy(), init_pose.astype(np.float32), cfg.match.dist_th)
        _t("refine", t0)
        aux["refine_rounds"] = rounds
    else:
        pose = init_pose
    aux.update(ss=ss_cat.numpy(), tt=tt_cat.numpy(), R_cat=R_cat.numpy(), t_cat=t_cat.numpy())
    return pose, num_inliers, num_mutual, len(inlier_ind), scales_used, aux


# --------------------------------------------------------------------------- #
# a17 / a18: baseline semantics of the reference's dead CPU modules (cpp_wrappers)
# --------------------------------------------------------------------------- #
def radius_neighbors(queries, supports, q_batches, s_batches, radius: float) -> np.ndarray:
    queries, supports = _f32(queries), _f32(supports)
    qb = np.ascontiguousarray(q_batches, dtype=np.int32)
    sb = np.ascontiguousarray(s_batches, dtype=np.int32)
    L = lib()
    L.bxo_radius_neighbors.argtypes = [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_float, c_void_p]
    L.bxo_free.argtypes = [c_void_p]
    out = c_void_p()
    mc = L.bxo_radius_neighbors(_p(queries), queries.shape[0], _p(supports), supports.shape[0], _p(qb), len(qb), _p(sb), len(sb),
                                c_float(radius), ctypes.byref(out))
    nq = queries.shape[0]
    arr = np.ctypeslib.as_array(ctypes.cast(out, POINTER(c_int32)), shape=(max(nq * mc, 1),))[: nq * mc].reshape(nq, mc).copy()
    L.bxo_free(out)
    return arr


def grid_subsample(points, dl: float):
    """-> (keys uint64 [m], barycentres fp32 [m,3], counts int32 [m]) in ascending cell-key order."""
    points = _f32(points)
    n = points.shape[0]
    keys = np.zeros(max(n, 1), dtype=np.uint64)
    xyz = np.zeros((max(n, 1), 3), dtype=np.float32)
    cnt = np.zeros(max(n, 1), dtype=np.int32)
    L = lib()
    L.bxo_grid_subsample.argtypes = [c_void_p, c_int, c_float, c_void_p, c_void_p, c_void_p]
    m = L.bxo_grid_subsample(_p(points), n, c_float(dl), _p(keys), _p(xyz), _p(cnt))
    return keys[:m].copy(), xyz[:m].copy(), cnt[:m].copy()


_REF_SO = os.path.join(_HERE, "_ref", "libbxref.so")


def ref_available() -> bool:
    return os.path.exists(_REF_SO)


_ref = None


def ref_lib():
    """The reference's own cpp_wrappers sources compiled unmodified (oracle/ref_build/build_ref.py)."""
    global _ref
    if _ref is None:
        _ref = ctypes.CDLL(_REF_SO)
        _ref.ref_batch_neighbors.argtypes = [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_float, c_void_p]
        _ref.ref_grid_subsampling.argtypes = [c_void_p, c_int, c_float, c_void_p]
        _ref.ref_free.argtypes = [c_void_p]
    return _ref


def ref_radius_neighbors(queries, supports, q_batches, s_batches, radius: float) -> np.ndarray:
    queries, supports = _f32(queries), _f32(supports)
    qb = np.ascontiguousarray(q_batches, dtype=np.int32)
    sb = np.ascontiguousarray(s_batches, dtype=np.int32)
    out = c_void_p()
    mc = ref_lib().ref_batch_neighbors(_p(queries), queries.shape[0], _p(supports), supports.shape[0], _p(qb), len(qb), _p(sb), len(sb),
                                       c_float(radius), ctypes.byref(out))
    nq = queries.shape[0]
    arr = np.ctypeslib.as_array(ctypes.cast(out, POINTER(c_int32)), shape=(max(nq * mc, 1),))[: nq * mc].reshape(nq, mc).copy()
    ref_lib().ref_free(out)
    return arr


def ref_grid_subsampling(points, dl: float) -> np.ndarray:
    points = _f32(points)
    out = c_void_p()
    m = ref_lib().ref_grid_subsampling(_p(points), points.shape[0], c_float(dl), ctypes.byref(out))
    arr = np.ctypeslib.as_array(ctypes.cast(out, POINTER(c_float)), shape=(max(3 * m, 1),))[: 3 * m].reshape(m, 3).copy()
    ref_lib().ref_free(out)
    return arr


# --------------------------------------------------------------------------- #
# SURVEY 8(f) row 1: loader-side geometric bootstrapping (float64 NumPy restatements)
# --------------------------------------------------------------------------- #
def pca_alignment(pts, sample_idx):
    """compute_pca_alignment (/root/reference/utils/tools.py:132-149) with the random sample made explicit.
    sklearn.decomposition.PCA(n_components=3).fit(X) on [n,3] float64 data: explained_variance_ = eigenvalues of the
    centred sample covariance (1/(n-1)), descending; components_ = eigenvectors as rows, each signed so that its entry of
    largest magnitude is positive (sklearn >= 1.5: svd_flip(u_based_decision=False)).  Pinned against sklearn itself in
    tests/test_oracle_cpu.py.  Returns (sphericity, is_aligned, mean, variance[3], components[3,3])."""
    X = np.asarray(pts, dtype=np.float64)[np.asarray(sample_idx)]
    if X.shape[0] < 3:                 # sklearn's PCA(n_components=3) refuses fewer samples than components
        raise ValueError(f"n_components=3 must be between 0 and min(n_samples, n_features)={X.shape[0]}")
    mean = X.mean(axis=0)
    Xc = X - mean
    C = (Xc.T @ Xc) / (X.shape[0] - 1)
    w, V = np.linalg.eigh(C)
    order = np.argsort(w)[::-1]
    w, V = w[order], V[:, order]
    comps = V.T.copy()
    for r in range(3):
        if comps[r, np.argmax(np.abs(comps[r]))] < 0:
            comps[r] = -comps[r]
    sphericity = w[2] / w[0]
    z = comps[2] / np.linalg.norm(comps[2])
    is_aligned = bool(abs(float(np.dot(z, np.array([0.0, 0.0, 1.0])))) > 0.98)
    return float(sphericity), is_aligned, mean, w, comps


def sphericity_based_voxel_analysis(src, tgt, idx_src, idx_tgt):
    """/root/reference/utils/tools.py:152-198 -> (voxel_size, sphericity, is_aligned_to_global_z)."""
    s_s, a_s, m_s, _, c_s = pca_alignment(src, idx_src)
    s_t, a_t, m_t, _, c_t = pca_alignment(tgt, idx_tgt)
    if len(src) > len(tgt):
        ref, sph, mean, comps = src, s_s, m_s, c_s
    else:
        ref, sph, mean, comps = tgt, s_t, m_t, c_t
    zt = (np.asarray(ref, dtype=np.float64) - mean) @ comps[2]
    z_range = zt.max() - zt.min()
    alpha = 1.0 if sph < 0.05 else 1.5
    voxel = max(np.sqrt(z_range) / 100 * alpha, 0.001)
    zs, zg = c_s[2] / np.linalg.norm(c_s[2]), c_t[2] / np.linalg.norm(c_t[2])
    same = float(np.dot(zs, zg)) > 0.96
    return round(float(voxel), 4), sph, bool(a_s and a_t and same)


def voxel_down_sample(pts, voxel: float):
    """open3d.geometry.PointCloud.voxel_down_sample (Open3D 0.18.0, cpp/open3d/geometry/PointCloud.cpp VoxelDownSample;
    not under /root/reference -- restated from the published algorithm, anchored on the call sites dataset/*.py and
    utils/tools.py:218-219): voxel_min_bound = min_bound - voxel*0.5; index = floor((p - voxel_min_bound)/voxel);
    output = mean of the points of a voxel (double accumulation).  Returns (keys [m] = ix | iy<<21 | iz<<42 sorted
    ascending, means [m,3] float64, counts [m]) -- Open3D's own output order is that of an unordered_map.  Like
    ops.voxel_down_sample it refuses a cloud spanning 2^21 voxels or more on an axis, where those keys would alias."""
    P = np.asarray(pts, dtype=np.float64)
    if not np.isfinite(P).all():
        raise ValueError("voxel_down_sample: needs finite coordinates")
    vmb = P.min(axis=0) - voxel * 0.5
    iv = np.floor((P - vmb) / voxel).astype(np.int64)
    if iv.max() >= 1 << 21:
        raise ValueError(f"voxel_down_sample: the cloud spans {iv.max() + 1} voxels of {voxel} on an axis; keys hold "
                         f"fewer than 2^21 = {1 << 21} per axis")
    keys = (iv[:, 0] & 0x1FFFFF) | ((iv[:, 1] & 0x1FFFFF) << 21) | ((iv[:, 2] & 0x1FFFFF) << 42)
    uk, inv, cnt = np.unique(keys, return_inverse=True, return_counts=True)
    sums = np.zeros((len(uk), 3))
    np.add.at(sums, inv, P)
    return uk, sums / cnt[:, None], cnt
