"""H100 drop-in for ``torch_batch_svd``: ``svd(A [B,3,3]) -> (U, S, V)`` with A = U diag(S) V^T and S descending, the
only form the BUFFER-X reference uses (utils/common.py:715, cal_Z_axis), on bufferx_b200's ``bx_svd3`` kernel (fp64
one-sided Jacobi, one thread per matrix, float32 out), forward only.  General matrices, not only symmetric ones.  Signs
of singular vectors are unspecified, as with the cuSOLVER original.  Needs the repository root on ``sys.path`` as well.
"""
import torch

from bufferx_b200 import ops

__all__ = ["svd"]


def svd(A):
    if isinstance(A, torch.Tensor) and (A.dim() != 3 or tuple(A.shape[1:]) != (3, 3)):
        raise NotImplementedError(f"torch_batch_svd.svd: only float32 [B,3,3] inputs are supported, got {tuple(A.shape)}")
    A = ops.dropin_tensor(A, "A", "[B,3,3]")
    with torch.cuda.device(A.device):
        return ops.svd3(A)
