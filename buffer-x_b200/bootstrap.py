"""GPU mirror of the reference's loader-side geometric bootstrapping (SURVEY.md 8(f) row 1).

Lives INSIDE the package (``bufferx_b200.bootstrap``), not in a top-level ``utils/`` directory: the reference's
``utils`` is a namespace package (no ``__init__.py``) and a regular ``utils`` package ahead of it on ``sys.path`` would
hide ``utils.timer`` / ``utils.SE3`` / ... from the reference's ``test.py`` (INTEGRATION.md section 1).

``sphericity_based_voxel_analysis`` keeps the reference's name, argument order and return tuple
(/root/reference/utils/tools.py:152-198); clouds are [N,3] arrays / CUDA tensors (or objects with a ``.points``
attribute, like the reference's Open3D clouds).  ``voxel_down_sample`` replaces
``open3d.geometry.PointCloud.voxel_down_sample`` at the call sites in dataset/*.py.  The arithmetic runs in
bx_pca_analysis / bx_project_range / bx_voxel_down_sample (csrc/bx_bootstrap.cu); there is no CPU fallback.
"""
import math

import numpy as np
import torch

from bufferx_b200 import ops


def _cloud(x, device, dtype=torch.float32):
    """An Open3D-like cloud (``.points``), array or tensor -> contiguous [N,3] `dtype` tensor on `device`."""
    if hasattr(x, "points"):
        x = np.asarray(x.points)
    if not isinstance(x, torch.Tensor):
        x = torch.from_numpy(np.ascontiguousarray(np.asarray(x), dtype=torch.empty((), dtype=dtype).numpy().dtype))
    return x.to(device=device, dtype=dtype).reshape(-1, 3).contiguous()


def compute_pca_alignment(pts: torch.Tensor, sample_idx=None):
    """-> (sphericity, is_aligned, (mean, variance, components) float64 CUDA tensors).  ``sample_idx``: the reference
    draws ``np.random.choice(N, N // 10, replace=False)`` from NumPy's global RNG (utils/tools.py:135-136); the same
    draw happens here when it is not given."""
    n = pts.shape[0]
    if sample_idx is None:
        sample_idx = np.random.choice(n, size=int(n / 10), replace=False)
    if not isinstance(sample_idx, torch.Tensor):
        sample_idx = torch.from_numpy(np.ascontiguousarray(sample_idx, dtype=np.int32))
    sample_idx = sample_idx.to(device=pts.device, dtype=torch.int32).contiguous()
    mean, var, comps = ops.pca_analysis(pts, sample_idx)
    h = torch.cat([var, comps[2]]).cpu().numpy()          # one small read: the decisions below are host decisions
    sphericity = float(h[2] / h[0])
    z = h[3:6] / np.linalg.norm(h[3:6])
    is_aligned = bool(abs(float(z[2])) > 0.98)
    return sphericity, is_aligned, (mean, var, comps)


def sphericity_based_voxel_analysis(src_pcd, tgt_pcd, sample_src=None, sample_tgt=None, device=None):
    """-> (voxel_size, sphericity, is_aligned_to_global_z), reference utils/tools.py:152-198."""
    device = device or torch.device("cuda", torch.cuda.current_device())
    src, tgt = _cloud(src_pcd, device), _cloud(tgt_pcd, device)
    s_s, a_s, (m_s, _, c_s) = compute_pca_alignment(src, sample_src)
    s_t, a_t, (m_t, _, c_t) = compute_pca_alignment(tgt, sample_tgt)
    if src.shape[0] > tgt.shape[0]:
        ref, sph, mean, comps = src, s_s, m_s, c_s
    else:
        ref, sph, mean, comps = tgt, s_t, m_t, c_t
    lo, hi = ops.project_range(ref, mean, comps[2]).cpu().tolist()
    z_range = hi - lo
    alpha = 1.0 if sph < 0.05 else 1.5
    voxel = max(math.sqrt(z_range) / 100 * alpha, 0.001)
    zs, zt = c_s[2].cpu().numpy(), c_t[2].cpu().numpy()
    same = float(np.dot(zs / np.linalg.norm(zs), zt / np.linalg.norm(zt))) > 0.96
    return round(voxel, 4), sph, bool(a_s and a_t and same)


def voxel_down_sample(pcd, voxel_size: float, device=None):
    """Mean point of every occupied voxel (Open3D semantics), [m,3] float32 CUDA tensor, voxels in ascending key order."""
    device = device or torch.device("cuda", torch.cuda.current_device())
    keys, xyz, _ = ops.voxel_down_sample(_cloud(pcd, device), float(voxel_size))
    return xyz[torch.argsort(keys)]
