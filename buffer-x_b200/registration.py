"""GPU point-to-point ICP with Open3D's interface: ``open3d.pipelines.registration.registration_icp`` as the reference's KITTI
loader calls it to refine every pair's ground-truth pose (/root/reference/dataset/kitti.py:95-102).

The loader adds one import and calls through it, with its arguments unchanged (INTEGRATION.md section 1)::

    from bufferx_b200 import registration as reg_icp
    reg = reg_icp.registration_icp(pcd0, pcd1, 0.20, np.eye(4),
                                   reg_icp.TransformationEstimationPointToPoint(),
                                   reg_icp.ICPConvergenceCriteria(max_iteration=200))

Clouds are Open3D-like objects (``.points``), [N,3] arrays or CUDA tensors, used in float64 as Open3D does.  The whole
iteration loop runs on the device (csrc/bx_icp.cu, the contract is written out there); the result is read once.  Where
Open3D defers to FLANN two rules are assumptions: the radius test is strict (d2 < r*r) and the lowest target index wins a
tie.  ``correspondence_set`` is sorted by source index (Open3D's order depends on its OpenMP threads).  There is no CPU
fallback: without a CUDA device the call raises.
"""
import numpy as np
import torch

from bufferx_b200 import ops
from bufferx_b200.bootstrap import _cloud


class TransformationEstimationPointToPoint:
    def __init__(self, with_scaling=False):
        self.with_scaling = bool(with_scaling)


class ICPConvergenceCriteria:
    def __init__(self, relative_fitness=1e-6, relative_rmse=1e-6, max_iteration=30):
        self.relative_fitness = float(relative_fitness)
        self.relative_rmse = float(relative_rmse)
        self.max_iteration = int(max_iteration)


class RegistrationResult:
    """transformation [4,4] float64, fitness, inlier_rmse, correspondence_set [k,2] int32 (source, target) by source index;
    also iterations (updates applied) and converged (the relative criteria stopped the loop)."""

    def __init__(self, transformation, fitness, inlier_rmse, correspondence_set, iterations, converged):
        self.transformation = transformation
        self.fitness = fitness
        self.inlier_rmse = inlier_rmse
        self.correspondence_set = correspondence_set
        self.iterations = iterations
        self.converged = converged

    def __repr__(self):
        return (f"RegistrationResult with fitness={self.fitness:e}, inlier_rmse={self.inlier_rmse:e}, "
                f"and correspondence_set size of {len(self.correspondence_set)}")


def _npoints(x):
    if hasattr(x, "points"):
        x = x.points
    return int(np.prod(np.shape(x))) // 3 if not isinstance(x, torch.Tensor) else x.numel() // 3


def registration_icp(source, target, max_correspondence_distance, init=np.eye(4), estimation_method=None, criteria=None):
    """Open3D 0.18 registration_icp with TransformationEstimationPointToPoint on the GPU -> RegistrationResult.
    Open3D's argument names; estimation_method must be a TransformationEstimationPointToPoint (this module's or Open3D's):
    any other estimation (point-to-plane, colored, generalized) is refused rather than run as point-to-point."""
    est = estimation_method if estimation_method is not None else TransformationEstimationPointToPoint()
    criteria = criteria if criteria is not None else ICPConvergenceCriteria()
    if type(est).__name__ != "TransformationEstimationPointToPoint":
        raise NotImplementedError(f"registration_icp: only TransformationEstimationPointToPoint is supported, got {type(est).__name__}")
    if getattr(est, "with_scaling", False):
        raise NotImplementedError("registration_icp: with_scaling=True is not supported (rigid point-to-point only)")
    r = float(max_correspondence_distance)
    if not r > 0.0:
        raise ops.BufferXError(f"registration_icp: max_correspondence_distance must be positive, got {r}")
    if _npoints(source) == 0 or _npoints(target) == 0:
        raise ops.BufferXError("registration_icp: empty source or target cloud")
    T0 = np.asarray(init.cpu() if isinstance(init, torch.Tensor) else init, dtype=np.float64)
    if T0.shape != (4, 4):
        raise ops.BufferXError(f"registration_icp: init must be 4x4, got {T0.shape}")
    if not torch.cuda.is_available():
        raise ops.BufferXError("registration_icp: no CUDA device (bufferx_b200 has no CPU path)")
    device = torch.device("cuda", torch.cuda.current_device())
    src = _cloud(source, device, torch.float64)
    tgt = _cloud(target, device, torch.float64)
    T0d = torch.from_numpy(np.ascontiguousarray(T0)).to(device)
    result, corr = ops.icp(src, tgt, r, T0d, criteria.relative_fitness, criteria.relative_rmse, criteria.max_iteration)
    T, fitness, rmse, _, iterations, converged = ops.decode_icp_result(result.cpu())
    c = corr[: src.shape[0]].cpu().numpy()
    idx = np.nonzero(c >= 0)[0]
    cs = np.stack([idx.astype(np.int32), c[idx]], axis=1) if len(idx) else np.zeros((0, 2), np.int32)
    return RegistrationResult(T, fitness, rmse, cs, iterations, converged)
