"""``pointnet2_ops.pointnet2_utils`` on bufferx_b200's sm_90a kernels, forward only.

    furthest_point_sample(xyz [B,N,3], npoint)         -> int32 [B,npoint]      bx_fps, in launches of <= 16 clouds
    gather_operation(features [B,C,N], idx [B,M])      -> [B,C,M]               bx_gather_channels
    ball_query(radius, nsample, xyz [B,N,3], new_xyz [B,M,3]) -> int32 [B,M,nsample]   bx_ball_query_batched
    grouping_operation(features [B,C,N], idx [B,M,S])  -> [B,C,M,S]             bx_gather_channels

Tensors are float32 / int32 CUDA tensors; every op runs on its inputs' device and that device's current stream.  CPU
tensors raise ``BufferXError``; inputs that require grad raise ``NotImplementedError`` (no backward is built).
"""
import torch

from bufferx_b200 import ops
from bufferx_b200.ops import BufferXError

__all__ = ["furthest_point_sample", "gather_operation", "ball_query", "grouping_operation"]

_FPS_CLOUDS = 16   # clouds per bx_fps launch


def furthest_point_sample(xyz, npoint):
    """Indices [B,npoint] int32 of the farthest point sampling of each cloud, starting at point 0."""
    xyz = ops.dropin_tensor(xyz, "xyz", "[B,N,3]")
    B, N, _ = xyz.shape
    npoint = int(npoint)
    with torch.cuda.device(xyz.device):
        parts = []
        for b0 in range(0, B, _FPS_CLOUDS):
            nb = min(_FPS_CLOUDS, B - b0)
            idx, _ = ops.fps(xyz[b0:b0 + nb].reshape(-1, 3), [b * N for b in range(nb + 1)], npoint, want_kpts=False)
            parts.append(idx)
        if not parts:
            return torch.empty((0, npoint), dtype=torch.int32, device=xyz.device)
        return parts[0] if len(parts) == 1 else torch.cat(parts)


def gather_operation(features, idx):
    """out[b,c,m] = features[b,c,idx[b,m]]."""
    features = ops.dropin_tensor(features, "features", "[B,C,N]")
    idx = ops.dropin_tensor(idx, "idx", "[B,M]", torch.int32)
    if idx.shape[0] != features.shape[0]:
        raise BufferXError(f"gather_operation: batch sizes differ: features {tuple(features.shape)}, idx {tuple(idx.shape)}")
    with torch.cuda.device(features.device):
        return ops.gather_channels(features, idx)


def ball_query(radius, nsample, xyz, new_xyz):
    """For every centre of new_xyz, the first nsample points of its cloud (index order) with squared distance
    < radius^2, padded with the first hit; an all-zero row when none is hit."""
    xyz = ops.dropin_tensor(xyz, "xyz", "[B,N,3]")
    new_xyz = ops.dropin_tensor(new_xyz, "new_xyz", "[B,M,3]")
    if new_xyz.shape[0] != xyz.shape[0] or xyz.shape[2] != 3 or new_xyz.shape[2] != 3:
        raise BufferXError(f"ball_query: expected xyz [B,N,3] and new_xyz [B,M,3], got {tuple(xyz.shape)} and {tuple(new_xyz.shape)}")
    with torch.cuda.device(xyz.device):
        return ops.ball_query_batched(xyz, new_xyz, float(radius), int(nsample))


def grouping_operation(features, idx):
    """out[b,c,m,s] = features[b,c,idx[b,m,s]]."""
    features = ops.dropin_tensor(features, "features", "[B,C,N]")
    idx = ops.dropin_tensor(idx, "idx", "[B,M,S]", torch.int32)
    if idx.shape[0] != features.shape[0]:
        raise BufferXError(f"grouping_operation: batch sizes differ: features {tuple(features.shape)}, idx {tuple(idx.shape)}")
    with torch.cuda.device(features.device):
        return ops.gather_channels(features, idx)
