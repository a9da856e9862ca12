"""bufferx_b200.registration refuses, before any launch, what it does not run: another estimation method, with_scaling,
r <= 0, empty clouds, a malformed init, and any call without a CUDA device; ops.icp refuses malformed tensors.  No GPU
needed."""
import numpy as np
import pytest
import torch

import bufferx_b200 as bx
from bufferx_b200 import registration as reg_icp

PTS = np.random.default_rng(0).uniform(-1, 1, (50, 3))


def test_defaults_match_open3d():
    c = reg_icp.ICPConvergenceCriteria()
    assert (c.relative_fitness, c.relative_rmse, c.max_iteration) == (1e-6, 1e-6, 30)
    assert reg_icp.TransformationEstimationPointToPoint().with_scaling is False


def test_with_scaling_is_refused():
    with pytest.raises(NotImplementedError):
        reg_icp.registration_icp(PTS, PTS, 0.2, np.eye(4), reg_icp.TransformationEstimationPointToPoint(with_scaling=True))


@pytest.mark.parametrize("r", [0.0, -0.2, float("nan")])
def test_nonpositive_radius_is_refused(r):
    with pytest.raises(bx.ops.BufferXError):
        reg_icp.registration_icp(PTS, PTS, r)


def test_empty_clouds_are_refused():
    with pytest.raises(bx.ops.BufferXError):
        reg_icp.registration_icp(np.zeros((0, 3)), PTS, 0.2)
    with pytest.raises(bx.ops.BufferXError):
        reg_icp.registration_icp(PTS, np.zeros((0, 3)), 0.2)


def test_cpu_only_use_is_refused(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(bx.ops.BufferXError):
        reg_icp.registration_icp(PTS, PTS, 0.2)


class TransformationEstimationPointToPlane:          # stands for Open3D's class of that name
    pass


class TransformationEstimationPointToPoint:          # an Open3D-like point-to-point estimation (by class name)
    with_scaling = False


def test_other_estimations_are_refused():
    for est in (TransformationEstimationPointToPlane(), object()):
        with pytest.raises(NotImplementedError):
            reg_icp.registration_icp(PTS, PTS, 0.2, np.eye(4), est)
        with pytest.raises(NotImplementedError):
            reg_icp.registration_icp(PTS, PTS, 0.2, estimation_method=est)


def test_open3d_like_point_to_point_is_accepted(monkeypatch):
    """An estimation of the right class name passes the estimation checks (and then stops at the CUDA check here)."""
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(bx.ops.BufferXError, match="no CUDA device"):
        reg_icp.registration_icp(PTS, PTS, 0.2, np.eye(4), TransformationEstimationPointToPoint())


def test_malformed_init_is_refused():
    with pytest.raises(bx.ops.BufferXError):
        reg_icp.registration_icp(PTS, PTS, 0.2, np.eye(3))


def test_ops_icp_checks_its_tensors():
    """ops.icp checks shapes before any launch: bx_icp reads 16 doubles of init and [N,3] clouds."""
    src = torch.zeros((5, 3), dtype=torch.float64)
    with pytest.raises(bx.ops.BufferXError, match="init"):
        bx.ops.icp(src, src, 0.2, torch.zeros((3, 4), dtype=torch.float64), 1e-6, 1e-6, 3)
    with pytest.raises(bx.ops.BufferXError, match="src"):
        bx.ops.icp(torch.zeros((5, 4), dtype=torch.float64), src, 0.2, torch.eye(4, dtype=torch.float64), 1e-6, 1e-6, 3)
